"""Host side of the tensor-core build kernel (dagr_l1_build_tc) without a GPU: the weight fragments dagr_l1a_tc_weights writes
are the [48][16] matrix (w[u][cin] at k = 3 u + cin, root[cin] at k = 45 + cin) in m16n8k8 B-fragment order, split into a
TF32 high part and an exact remainder; and the entry point refuses missing params / fragments before anything is launched."""
import ctypes as C

import numpy as np

E_ARG = -1


def _tf32_rna(x):
    """cvt.rna.tf32.f32 on finite values: round to nearest, ties away from zero, low 13 mantissa bits cleared."""
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + 0x1000) & 0xffffe000).astype(np.uint32).view(np.float32)


def _params(seed):
    from dagr_b200 import _lib
    g = np.random.default_rng(seed)
    w = (g.standard_normal((15, 3, 16)) * 0.3).astype(np.float32)
    root = (g.standard_normal((3, 16)) * 0.3).astype(np.float32)
    p = _lib.L1AParams()
    C.memmove(p.w, w.ctypes.data, w.nbytes)
    C.memmove(p.root, root.ctypes.data, root.nbytes)
    return p, w, root


def test_fragments_are_the_48x16_weight_matrix_in_b_fragment_order():
    from dagr_b200 import _lib
    lib = _lib.load()
    p, w, root = _params(5)
    out = (C.c_float * _lib.L1A_TC_WFRAG_FLOATS)()
    assert lib.dagr_l1a_tc_weights(C.byref(p), C.cast(out, C.c_void_p)) == 0
    f = np.frombuffer(out, dtype=np.float32).reshape(6, 32, 2, 4)           # [k-step][lane][n-tile](hi b0, hi b1, lo b0, lo b1)
    B = np.concatenate([w.reshape(45, 16), root], axis=0)                    # [k][n]
    s, lane, nt = np.meshgrid(np.arange(6), np.arange(32), np.arange(2), indexing="ij")
    gq, t = lane >> 2, lane & 3
    n = 8 * nt + gq
    b0, b1 = B[8 * s + t, n], B[8 * s + t + 4, n]
    h0, h1 = _tf32_rna(b0), _tf32_rna(b1)
    assert np.array_equal(f[..., 0], h0) and np.array_equal(f[..., 1], h1)
    assert np.array_equal(f[..., 2], b0 - h0) and np.array_equal(f[..., 3], b1 - h1)
    # the split is exact and the high parts are TF32 values
    assert np.array_equal(f[..., 0] + f[..., 2], b0) and np.array_equal(f[..., 1] + f[..., 3], b1)
    assert not (f[..., :2].view(np.uint32) & 0x1fff).any()


def test_tc_build_refuses_missing_params_or_fragments():
    from dagr_b200 import _lib
    lib = _lib.load()
    p, _, _ = _params(1)
    frag = (C.c_float * _lib.L1A_TC_WFRAG_FLOATS)()
    args = lambda params, wfrag: (None, 10, None, None, None, None, params, wfrag, None, 0, None, None, None, None, None, None, 0, None)
    for params, wfrag in ((C.byref(p), None), (None, C.cast(frag, C.c_void_p))):
        assert lib.dagr_l1_build_tc(*args(params, wfrag)) == E_ARG
        assert b"weight fragments" in lib.dagr_last_error()
    assert lib.dagr_l1a_tc_weights(None, C.cast(frag, C.c_void_p)) == E_ARG
    assert lib.dagr_l1a_tc_weights(C.byref(p), None) == E_ARG
