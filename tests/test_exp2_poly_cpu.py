"""rp_selftest_exp2 argument checks: decided before any CUDA call, so they run without a GPU."""


def test_selftest_exp2_argument_errors_without_a_gpu():
    import ctypes

    from replay_b200._lib import lib

    L = lib()
    EINVAL = -1
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert L.rp_selftest_exp2(None, p, p, 4, None) == EINVAL
    assert L.rp_selftest_exp2(p, None, p, 4, None) == EINVAL
    assert L.rp_selftest_exp2(p, p, None, 4, None) == EINVAL
    assert L.rp_selftest_exp2(p, p, p, -1, None) == EINVAL
    assert L.rp_selftest_exp2(p, p, p, 0, None) == 0          # nothing to do: no launch
