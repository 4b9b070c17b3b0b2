"""RefCheck's choice between the compiled reference and the stored digests when only part of oracle/_ref is built."""
import json

import numpy as np
import pytest

import cpulibs as cl


def test_missing_feature_library_takes_stored_digests(tmp_path, monkeypatch):
    """libffref.so built and the block's feature library not (a partial reference build): the block compares with the stored
    digests and never calls the reference, and a result that differs from them still fails"""
    (tmp_path / "libffref.so").write_bytes(b"")
    monkeypatch.setattr(cl, "REF_DIR", str(tmp_path))
    monkeypatch.setattr(cl, "REF_SO", str(tmp_path / "libffref.so"))
    assert cl.have_ref() and not cl.have_ref("libffref_absent")
    ours = [np.arange(12, dtype=np.int16).reshape(3, 4), 7]
    test = "test_refcheck.py::test_missing_feature_library_takes_stored_digests"
    digests = tmp_path / "digests.json"
    digests.write_text(json.dumps({f"{test}#0": cl.ref_digest(ours), f"{test}#1": cl.ref_digest(ours)}))

    def theirs():
        raise AssertionError("the block called the reference")
    with cl.RefCheck(str(digests), "libffref_absent") as rc:
        assert not rc.live
        assert rc.same(ours, theirs)
    with pytest.raises(AssertionError, match="differs from the stored reference results"):
        with cl.RefCheck(str(digests), "libffref_absent") as rc:
            rc.same([ours[0] + 1, 7], theirs)
