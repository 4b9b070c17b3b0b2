"""Writes tests/golden/hevcpred_hashes.txt from the compiled reference (oracle/_ref/libffref_hevcpred.so): per depth x luma / 4:2:0 /
4:2:2 / 4:4:4 x constrained intra prediction off / on, the hash of the reference's reconstructed plane (guard frame included) for
hevcpredlib.fixture_case.  The digests of tests/golden/hevcpred_ref_digests.json are written by the tests themselves:
FFDSP_RECORD_REF=1 python -m pytest tests/test_hevc_pred.py"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import hevcpredlib as hl  # noqa: E402

if __name__ == "__main__":
    assert hl.have_ref(), "build oracle/_ref/libffref_hevcpred.so first (oracle/ref/hevcpred.mk)"
    with open(hl.FIXTURE, "w") as f:
        for depth in hl.DEPTHS:
            for name in hl.FIXTURE_CFMT:
                for cip in (False, True):
                    f.write(f"{depth} {hl.fixture_key(name, cip)} {hl.digest(hl.ref_plane(hl.fixture_case(depth, name, cip)))}\n")
