"""Writes tests/golden/vp8dsp_hashes.txt from the compiled reference (oracle/_ref/libffref_vp8dsp.so): per (is_vp7, bilinear), the hash
of the reference driver's three planes after vp8dsplib.fixture_case's inter frame and then its residual; then runs tests/test_vp8_dsp.py
with FFDSP_RECORD_REF=1, which rewrites the digests of tests/golden/vp8dsp_ref_digests.json (through the shared cpulibs.RefCheck)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp8dsplib as v8  # noqa: E402

if __name__ == "__main__":
    assert v8.have_ref(), "build oracle/_ref/libffref_vp8dsp.so first (oracle/ref/vp8dsp.mk)"
    with open(v8.FIXTURE, "w") as f:
        for is_vp7, bil in v8.FIXTURE_CASES:
            refs, ops, dst, rops, coef = v8.fixture_case(is_vp7, bil)
            planes = v8.ref_residual_frame(is_vp7, rops, coef, v8.ref_mc_frame(bil, 12, 9, refs, ops, dst))
            f.write(f"{is_vp7} {bil} {v8.digest(planes)}\n")
    if os.path.exists(v8.REF_DIGESTS):
        os.remove(v8.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp8_dsp.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
