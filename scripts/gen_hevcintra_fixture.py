"""Writes tests/golden/hevcintra_hashes.txt from the compiled reference (oracle/_ref/libffref_hevcintra.so): per fixture picture of
hevcintralib.FIXTURES, the hash of the framed planes (sentinels included) after the reference's intra_pred and residual sequence TU by
TU in decode order; then runs tests/test_hevc_intra_recon.py with FFDSP_RECORD_REF=1, which rewrites the digests of
tests/golden/hevcintra_ref_digests.json."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import hevcintralib as hl  # noqa: E402

if __name__ == "__main__":
    assert hl.have_ref(), "build oracle/_ref/libffref_hevcintra.so first (oracle/ref/hevcintra.mk)"
    with open(hl.FIXTURE, "w") as out:
        for name in hl.FIXTURE_NAMES:
            out.write(f"{name} {hl.digest(hl.ref_picture(hl.fixture_case(name)))}\n")
    if os.path.exists(hl.REF_DIGESTS):
        os.remove(hl.REF_DIGESTS)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "not gpu", os.path.join(ROOT, "tests", "test_hevc_intra_recon.py")],
                   env=dict(os.environ, FFDSP_RECORD_REF="1"), cwd=ROOT, check=True)
