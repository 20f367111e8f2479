"""The inertialization entry points through the C ABI without a device: a NULL context (and, for the decodes, a NULL clip set) is refused
with ACLB200_ERR_INVALID_ARGUMENT before anything else is read, and the request records have the header's layout. The refusals that need
a context are in tests/test_gpu_inertialization.py."""
import ctypes as C

import numpy as np

INVALID_ARGUMENT = 1


def test_null_context_is_refused():
    import acl_b200 as ab
    from acl_b200 import api
    lib = api._lib()
    options = ab.Options()
    assert lib.aclb200_begin_inertialization(None, None, None, None, None, 4, 3, 0, 30.0, None, 0, None, None) == INVALID_ARGUMENT
    assert lib.aclb200_inertialize_poses(None, None, None, 4, 3, 0, None, None, 1, 0, None) == INVALID_ARGUMENT
    assert lib.aclb200_decompress_tracks_inertialized(None, None, None, 4, C.byref(options), None, 0, 0, None, None, 0, None, None,
                                                      None) == INVALID_ARGUMENT
    assert lib.aclb200_decompress_tracks_inertialized_skinning(None, None, None, 4, C.byref(options), None, 0, 0, None, None, None, None,
                                                               None, None) == INVALID_ARGUMENT


def test_record_layouts():
    """aclb200_inertialization is 12 bytes and aclb200_inertialized_request 20 (a request, then its inertialization); the helpers fill
    every field and broadcast"""
    import acl_b200 as ab
    assert ab.INERTIALIZATION_DTYPE.itemsize == 12
    assert ab.INERTIALIZED_REQUEST_DTYPE.itemsize == 20
    assert ab.INERTIALIZED_REQUEST_DTYPE.fields["record"][1] == 8
    r = ab.make_inertialized_requests([3, 4], 0.5, [ab.NO_INERTIALIZATION, 7], 0.25, 0.1)
    words = r.view(np.uint32).reshape(2, 5)
    assert words[:, 0].tolist() == [3, 4] and words[:, 2].tolist() == [0xFFFFFFFF, 7]
    assert words[:, 1].view(np.float32).tolist() == [0.5, 0.5] and words[:, 4].view(np.float32).tolist() == [np.float32(0.1)] * 2
    i = ab.make_inertializations([1, 2, 3], 0.0, 0.2)
    assert i.view(np.uint32).reshape(3, 3)[:, 0].tolist() == [1, 2, 3]
