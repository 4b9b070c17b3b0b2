"""Writes tests/golden/vp9lf_hashes.txt from the compiled reference (oracle/_ref/libffref_vp9lf.so): per depth x chroma format x record
kind, the hash of the reference driver's three planes (sentinels included) after ff_vp9_loopfilter_sb over vp9lflib.frame_case in raster
order; then runs tests/test_vp9_loopfilter.py with FFDSP_RECORD_REF=1, which rewrites the digests of tests/golden/vp9lf_ref_digests.json."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp9lflib as vl  # noqa: E402

if __name__ == "__main__":
    assert vl.have_ref(), "build oracle/_ref/libffref_vp9lf.so first (oracle/ref/Makefile)"
    with open(vl.FIXTURE, "w") as f:
        for name in vl.FIXTURE_NAMES:
            f.write(f"{name} {vl.digest(vl.ref_frame(vl.frame_case(name)))}\n")
    if os.path.exists(vl.REF_DIGESTS):
        os.remove(vl.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp9_loopfilter.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
