"""Writes tests/golden/vp9intra_hashes.txt from the compiled reference (oracle/_ref/libffref_vp9intra.so): per fixture frame of
vp9intralib.FIXTURES, the hash of the three planes (sentinels included) after the reference's intra_recon block by block, run with tight
line sizes (the emulated-edge path) and again with wide ones, which must agree; then runs tests/test_vp9_intra.py with FFDSP_RECORD_REF=1,
which rewrites the digests of tests/golden/vp9intra_ref_digests.json."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp9intralib as vi  # noqa: E402

if __name__ == "__main__":
    assert vi.have_ref(), "build oracle/_ref/libffref_vp9intra.so first (oracle/ref/Makefile)"
    with open(vi.FIXTURE, "w") as out:
        for name in vi.FIXTURE_NAMES:
            f = vi.frame_case(name)
            tight, wide = vi.ref_frame(f, tight=True), vi.ref_frame(f)
            assert all(np.array_equal(a, b) for a, b in zip(tight, wide)), name
            full = [p.copy() for p in f.planes]
            for a, r in zip(f.area(full), tight):
                a[...] = r
            out.write(f"{name} {vi.digest(full)}\n")
    if os.path.exists(vi.REF_DIGESTS):
        os.remove(vi.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_vp9_intra.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
