"""Writes tests/golden/vp9mc_hashes.txt from the compiled reference (oracle/_ref/libffref_vp9dsp.so): per depth x luma- / 4:2:0-chroma-
shaped plane, the hash of the reference driver's destination picture (sentinels included) for vp9mclib.fixture_case; then runs
tests/test_vp9_mc.py with FFDSP_RECORD_REF=1, which rewrites the digests of tests/golden/vp9mc_ref_digests.json."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp9mclib as vm  # noqa: E402

if __name__ == "__main__":
    assert vm.have_ref(), "build oracle/_ref/libffref_vp9dsp.so first (oracle/ref/Makefile)"
    with open(vm.FIXTURE, "w") as f:
        for depth in vm.DEPTHS:
            for chroma in (0, 1):
                f.write(f"{depth} {'chroma' if chroma else 'luma'} {vm.digest(vm.ref_batch(depth, *vm.fixture_case(depth, chroma)))}\n")
    if os.path.exists(vm.REF_DIGESTS):
        os.remove(vm.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp9_mc.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
