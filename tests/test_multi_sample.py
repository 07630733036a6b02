"""MultiLLM.sample_many, host side: how its settings are spread over the slots (multi.per_slot), and the refusals of the C entry
points that need no device."""
import ctypes as C

import numpy as np
import pytest

from ctransformers_b200.multi import per_slot


def test_one_value_is_every_slots():
    assert per_slot(40, 3, "top_k") == [40, 40, 40]
    assert per_slot(0.95, 1, "top_p") == [0.95]
    assert per_slot(None, 2, "seed") == [None, None]
    assert per_slot(7, 0, "seed") == []


def test_a_sequence_is_one_value_per_slot():
    assert per_slot([1, 40, 0], 3, "top_k") == [1, 40, 0]
    assert per_slot((0.5, None), 2, "top_p") == [0.5, None]          # None: that slot takes the config's value
    assert per_slot(np.array([1.1, 1.3], np.float32), 2, "repetition_penalty") == pytest.approx([1.1, 1.3])
    assert per_slot(range(4), 4, "seed") == [0, 1, 2, 3]


@pytest.mark.parametrize("value, n", [([1, 2], 3), ([1, 2, 3, 4], 3), ([], 1), ([5], 0)])
def test_wrong_length_is_refused(value, n):
    with pytest.raises(ValueError, match="top_k"):
        per_slot(value, n, "top_k")


def test_rows_ops_refuse_bad_arguments_without_launching(lib):
    """No rows, rows of no logits and descending window offsets are refused before anything reaches a device."""
    x = np.zeros(8, np.float32)
    ip = lambda v: (C.c_int * max(len(v), 1))(*v)
    fp = lambda v: (C.c_float * max(len(v), 1))(*v)
    out = np.zeros(2 * 256, np.int32)
    o = out.ctypes.data_as(C.POINTER(C.c_int))
    lg = np.zeros(2 * 256, np.float32).ctypes.data_as(C.POINTER(C.c_float))
    for n_rows, n, off in ((0, 4, [0]), (2, 0, [0, 0, 0]), (2, 4, [0, 3, 1])):
        assert lib.ctb_sample_topk_rows(x.ctypes.data_as(C.c_void_p), n_rows, n, ip(off), ip([1, 2, 3]), fp([1.0, 1.0]), ip([1, 1]), o, o, lg) == -1
        assert lib.ctb_sample_device_rows(x.ctypes.data_as(C.c_void_p), n_rows, n, ip(off), ip([1, 2, 3]), ip([1, 1]), fp([1.0, 1.0]),
                                          fp([1.0, 1.0]), fp([1.0, 1.0]), ip([0, 0]), o, o) == -1
