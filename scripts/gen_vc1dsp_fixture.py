"""Writes tests/golden/vc1dsp_hashes.txt from the compiled reference (oracle/_ref/libffref_vc1dsp.so): per vc1dsplib.FIXTURE_CASES entry,
the hash of the reference driver's three planes after the decoder-shaped picture's MC and then its residual; then runs
tests/test_vc1_dsp.py with FFDSP_RECORD_REF=1, which rewrites the digests of tests/golden/vc1dsp_ref_digests.json (through the shared
cpulibs.RefCheck)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vc1dsplib as v1  # noqa: E402

if __name__ == "__main__":
    assert v1.have_ref(), "build oracle/_ref/libffref_vc1dsp.so first (oracle/ref/vc1dsp.mk)"
    with open(v1.FIXTURE, "w") as f:
        for case in v1.FIXTURE_CASES:
            mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(case[0])
            planes = v1.ref_residual_frame(mbw, mbh, rops, coef, v1.ref_mc_frame(mbw, mbh, H, V, refs, ops, dst))
            f.write(f"{case[0]} {v1.digest(planes)}\n")
    if os.path.exists(v1.REF_DIGESTS):
        os.remove(v1.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vc1_dsp.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
