"""CPU checks of the planted rows that expose the order of the norms' fp64 sums (refs.norm_order_rows).  The numpy restatement
of both norms in the reference's order must equal the oracle bit for bit on every row, and the kernels' order
(refs.kernel_order_sum) must change the float statistic and the output at every thread count a build can give the kernels:
otherwise the GPU tests on these rows would pass on a kernel that sums in its own order."""
import numpy as np
import pytest

import refs
from conftest import ptr

KS = [256, 512, 1024, 4096, 4544, 4608, 8192, 11008]   # one partial warp .. several passes; 4544 / 11008 not multiples of NT·16


def _oracle_norm(mode, x, w, b, eps):
    o = refs.oracle()
    y = np.zeros_like(x)
    for i in range(x.shape[0]):
        if mode == 1:
            o.orc_rms_norm_mul(ptr(x[i]), ptr(w), ptr(y[i]), x.shape[1], eps)
        else:
            o.orc_layer_norm_mul_add(ptr(x[i]), ptr(w), ptr(b), ptr(y[i]), x.shape[1], eps)
    return y


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", [1, 2])
def test_sequential_restatement_is_the_oracle(mode, k):
    rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
    gauss = np.random.default_rng(k).standard_normal((4, k)).astype(np.float32) * np.float32(3)
    x = np.ascontiguousarray(np.concatenate([rows, gauss]))
    want = _oracle_norm(mode, x, w, b, refs.NORM_ORDER_EPS)
    got, _ = refs.norm_emulated(mode, x, w, b, refs.NORM_ORDER_EPS, refs.seq_sum)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", [1, 2])
def test_kernel_order_changes_every_row(mode, k):
    rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
    y_ref, st_ref = refs.norm_emulated(mode, rows, w, b, refs.NORM_ORDER_EPS, refs.seq_sum)
    for nt in refs.NORM_ORDER_THREADS:
        y, st = refs.norm_emulated(mode, rows, w, b, refs.NORM_ORDER_EPS, lambda t: refs.kernel_order_sum(t, nt))
        assert (y.view(np.uint32) != y_ref.view(np.uint32)).any(axis=1).all(), nt
        if mode == 1:
            assert (st[0] != st_ref[0]).all(), nt
        else:   # rows 0-3 break Σx; rows 4-7 have Σx = 0 in both orders and break Σ(x - mean)² alone
            assert (st[0][:4] != st_ref[0][:4]).all() and (st[0][4:] == 0).all() and (st_ref[0][4:] == 0).all(), nt
            assert (st[1][4:] != st_ref[1][4:]).all(), nt


def test_kernel_order_sum_restates_the_thread_chains():
    """kernel_order_sum against a plain loop over threads, lanes and warps, on terms of wildly different sizes."""
    rng = np.random.default_rng(7)
    K, nt = 3000, 96
    t = np.ldexp(rng.uniform(1, 2, K), rng.integers(-60, 0, K))
    passes = -(-K // (nt * 16))
    lanes = []
    for th in range(nt):
        s = 0.0
        for ps in range(passes):
            for e in range(16):
                i = (ps * nt + th) * 16 + e
                if i < K:
                    s += t[i]
        lanes.append(s)
    warps = []
    for w in range(nt // 32):
        v = lanes[32 * w:32 * w + 32]
        for o in (16, 8, 4, 2, 1):
            v = [v[i] + v[i ^ o] for i in range(32)]
        warps.append(v[0])
    total = 0.0
    for s in warps:
        total += s
    assert refs.kernel_order_sum(t, nt) == total
