"""Writes tests/golden/vp8lf_hashes.txt from the compiled reference (oracle/_ref/libffref_vp8lf.so): per codec x filter type x
keyframe x record kind, the hash of the three planes (sentinels included) after the reference members in the decoder's raster sequence
over vp8lflib.frame_case; then runs tests/test_vp8_loopfilter.py with FFDSP_RECORD_REF=1, which rewrites the digests of
tests/golden/vp8lf_ref_digests.json."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp8lflib as vl  # noqa: E402

if __name__ == "__main__":
    assert vl.have_ref(), "build oracle/_ref/libffref_vp8lf.so first (oracle/ref/vp8lf.mk)"
    with open(vl.FIXTURE, "w") as f:
        for name in vl.FIXTURE_NAMES:
            f.write(f"{name} {vl.digest(vl.ref_frame(vl.frame_case(name)))}\n")
    if os.path.exists(vl.REF_DIGESTS):
        os.remove(vl.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp8_loopfilter.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
