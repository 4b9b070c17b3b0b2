#!/usr/bin/env python
"""Writes tests/golden/pel_layout_ref_digests.json: the digests of the COMPILED REFERENCE's results (oracle/_ref/libffref.so) for the
cases of tests/test_oracle_pel_layouts.py, which then check the motion-compensation checker against them on machines without the
reference.  Runs that test file with FFDSP_RECORD_REF=1 from an empty digest file; every case is still compared live while recording.
Run where the reference is built: python scripts/gen_pel_layout_digests.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "pel_layout_ref_digests.json")

if __name__ == "__main__":
    assert os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libffref.so")), "build oracle/_ref/libffref.so first (__graft_entry__.build())"
    if os.path.exists(OUT):
        os.remove(OUT)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join("tests", "test_oracle_pel_layouts.py")],
                   cwd=ROOT, env=dict(os.environ, FFDSP_RECORD_REF="1"), check=True)
    print("wrote", OUT)
