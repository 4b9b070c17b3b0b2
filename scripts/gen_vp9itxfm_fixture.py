"""Writes tests/golden/vp9itxfm_hashes.txt from the compiled reference (oracle/_ref/libffref_vp9itxfm.so): per depth x coefficient
class, the hash of the reference driver's destination picture (sentinels included) for vp9itxfmlib.fixture_case; then runs
tests/test_vp9_itxfm.py with FFDSP_RECORD_REF=1, which rewrites the digests of tests/golden/vp9itxfm_ref_digests.json."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp9itxfmlib as vt  # noqa: E402

if __name__ == "__main__":
    assert vt.have_ref(), "build oracle/_ref/libffref_vp9itxfm.so first (oracle/ref/vp9itxfm.mk)"
    with open(vt.FIXTURE, "w") as f:
        for depth in vt.DEPTHS:
            for cls in vt.FIXTURE_CLASSES:
                f.write(f"{depth} {cls} {vt.digest(vt.ref_batch(depth, *vt.fixture_case(depth, cls)))}\n")
    if os.path.exists(vt.REF_DIGESTS):
        os.remove(vt.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp9_itxfm.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
