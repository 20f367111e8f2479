"""The mirror entry points through the C ABI without a device: a NULL context is refused with ACLB200_ERR_INVALID_ARGUMENT before anything
else is read, the mirror entry and the mirrored request have the header's layout, and the helpers fill every field. The refusals that need
a context are in tests/test_gpu_mirror.py."""
import ctypes as C

import numpy as np

INVALID_ARGUMENT = 1


def test_null_context_is_refused():
    import acl_b200 as ab
    from acl_b200 import api
    lib = api._lib()
    options = ab.Options()
    assert lib.aclb200_mirror_poses(None, None, None, 4, 3, 0, None, None, 0, None, None) == INVALID_ARGUMENT
    assert lib.aclb200_decompress_tracks_mirrored(None, None, None, 4, C.byref(options), None, 0, None, None, 0, None, None, None) == INVALID_ARGUMENT
    assert lib.aclb200_decompress_tracks_mirrored_skinning(None, None, None, 4, C.byref(options), None, 0, None, None, None, None, None,
                                                           None) == INVALID_ARGUMENT


def test_record_layouts():
    """aclb200_mirror_entry is 48 bytes (pre, post, mirror, three reserved words) and aclb200_mirrored_request 12 (a request, then its
    flag); the helpers fill every field and broadcast"""
    import acl_b200 as ab
    assert ab.MIRROR_ENTRY_DTYPE.itemsize == 48
    assert [ab.MIRROR_ENTRY_DTYPE.fields[f][1] for f in ("pre", "post", "mirror", "reserved")] == [0, 16, 32, 36]
    assert ab.MIRRORED_REQUEST_DTYPE.itemsize == 12 and ab.MIRRORED_REQUEST_DTYPE.fields["mirrored"][1] == 8
    assert (ab.MIRROR_X, ab.MIRROR_Y, ab.MIRROR_Z, ab.ERROR_FLAG_INVALID_MIRROR) == (0, 1, 2, 8)
    r = ab.make_mirrored_requests([3, 4], 0.5, [0, 1])
    words = r.view(np.uint32).reshape(2, 3)
    assert words[:, 0].tolist() == [3, 4] and words[:, 2].tolist() == [0, 1]
    assert words[:, 1].view(np.float32).tolist() == [0.5, 0.5]


def test_table_helpers_fill_every_field():
    import acl_b200 as ab
    from tests import mirror_cases as cases
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    table = ab.mirror_table(parents, mirror, rotations, ab.MIRROR_Y)
    assert table["mirror"].tolist() == mirror.tolist()
    assert (table["reserved"] == 0).all()
    np.testing.assert_allclose(np.linalg.norm(table["pre"], axis=1), 1.0, rtol=1e-6)
    # roots take the identity as post, other bones conj(C_parent)
    assert table["post"][0].tolist() == [0, 0, 0, 1]
    np.testing.assert_array_equal(table["post"][3], table["pre"][2] * np.float32([-1, -1, -1, 1]))
    rows = ab.mirror_rows_table(table, [3, 6, 1], 1)
    assert rows["mirror"].tolist() == [1, 0, 2] and (rows["reserved"] == 0).all()
    np.testing.assert_array_equal(rows["pre"], table["pre"][[3, 6, 1]])
    np.testing.assert_array_equal(rows["post"], np.tile(table["pre"][1] * np.float32([-1, -1, -1, 1]), (3, 1)))
