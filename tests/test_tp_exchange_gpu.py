"""GPU parity tests of the tensor-sharded mode's fused exchange on one GPU: the exchange build of the step kernel
(k_step<true, ...>, and k_step<true, false, true> for Q3_K programs) through ctb_xchg_mul_mat, one rank of a W-rank world at a
time, the peers' stores simulated by entries written before each launch (tests/tp_exchange_refs.py).  Bar: bit-exact against
oracle pieces: every consumer's outputs and summed input, every region's slots with their exchange numbers, the exchange
count the launches leave, and the build that ran."""
import functools

import numpy as np
import pytest

import refs
import tp_exchange_refs as X
from test_ops_gpu import _same_bits

pytestmark = pytest.mark.gpu

STEPS = 2


@functools.lru_cache(maxsize=None)
def _case(case):
    c = X.CASES[case]
    types, mats = X.model(c, seed=500 + len(case))
    attn, res0, norm_w, peers = X.inputs(c, seed=600 + len(case))
    return c, types, mats, attn, res0, norm_w, peers


def _check_ll(ll, want, me, world, n_layers, base, what):
    """ll [layer][region R][parity][slot r][n_embd][2] after the last launch: in every region this rank's slots of both parity
    halves hold its two producers' rows with the last launch's numbers; the peers' slots hold what was written for that launch
    in this rank's region and are still zero in the others."""
    n_x = 2 * n_layers
    last = (base + (STEPS - 1) * n_x) & 0xFFFFFFFF
    for k in range(n_x):
        e = (last + k + 1) & 0xFFFFFFFF
        half = ll[k // 2, :, e & 1]
        for R in range(world):
            for r in range(world):
                where = f"{what}: exchange {k}, region {R}, slot {r}"
                if r == me or R == me:
                    _same_bits(half[R, r, :, 0].view(np.float32), want["parts"][k][r], where)
                    assert (half[R, r, :, 1] == e).all(), f"{where}: numbers {np.unique(half[R, r, :, 1])[:4]} for {e}"
                else:
                    assert not half[R, r].any(), f"{where}: a slot no rank writes here changed"


def _run_and_check(lib, c, me, types, mats, attn, res0, norm_w, parts, want, base, what, n_layers=X.N_LAYERS, eps=1e-5):
    rc, out, sums, ll, sync2, launch = X.run(lib, c, me, types, mats, attn, res0, norm_w, parts, base, steps=STEPS, eps=eps, n_layers=n_layers)
    assert rc == 0, what
    q3 = int(X.Q3_K in types)
    assert launch == (1, q3, 1), f"{what}: launched {launch}, meant the exchange build, Q3_K build {q3}, one CTA per cluster"
    _same_bits(out, np.concatenate(want["outs"]), f"{what}: consumer outputs")
    _same_bits(sums, np.stack(want["sums"]), f"{what}: sum_out")
    assert sync2 == (base + 2 * n_layers * STEPS) & 0xFFFFFFFF, f"{what}: sync[2] = {sync2:#x}"
    _check_ll(ll, want, me, c[5], n_layers, base, what)


@pytest.mark.parametrize("case", list(X.CASES))
def test_exchange_build_bit_exact(lib, case):
    """Every rank of the case, two layers (both parity halves twice), two launches back to back, from exchange counts 0, a
    middle value and 0xFFFFFFFD (the numbers wrap past 0 inside the program): consumer outputs and sums, the regions, sync[2]
    and the launch, bit for bit.  Cases with own_peers take the peers' partials from the peers' own shards."""
    c, types, mats, attn, res0, norm_w, peers = _case(case)
    for me in c[6]:
        want = X.expected(c, me, types, mats, attn, res0, norm_w, peers)
        for base in X.BASES:
            _run_and_check(lib, c, me, types, mats, attn, res0, norm_w, want["parts"], want, base, f"{case} rank {me} base {base:#x}")


# width: (n_head, n_ff, world); head_dim 128
PLANTED = {1024: (8, 512, 2), 4096: (32, 1024, 4), 8192: (64, 2048, 8)}


@pytest.mark.parametrize("k", list(PLANTED))
def test_planted_norm_rows_through_the_exchange(lib, k):
    """The first consumer's RMSNorm on refs.norm_order_rows rows whose fp64 sum of squares rounds differently in the kernel's
    order (the element-order fallback of norm_stat, under x_mode 2): rank 0 of W runs one layer on a zero attention vector, so
    its P_wo rows are the residual, which holds the row's low significand bits; the peers hold the higher bits."""
    nh, F, W = PLANTED[k]
    c = (k, nh, nh, F, 272, W, (0,), "Q4_K_M", "random", False)
    types, mats = X.model(c, seed=k, n_layers=1)
    rows, w, _ = refs.norm_order_rows(1, k, seed=k + W)
    _, _, norm_w, peers = X.inputs(c, seed=k + 1, n_layers=1)
    norm_w[0] = w
    attn = np.zeros((1, k), np.float32)
    for i, x in enumerate(rows):
        split = X.split_mantissa(x, W)
        peers[0] = np.stack(split)
        want = X.expected(c, 0, types, mats, attn, split[0], norm_w, peers, eps=refs.NORM_ORDER_EPS, n_layers=1)
        _same_bits(want["sums"][0], x, "the planted row's split")
        _run_and_check(lib, c, 0, types, mats, attn, split[0], norm_w, want["parts"], want, X.BASES[i % 3], f"k {k} row {i}", n_layers=1,
                       eps=refs.NORM_ORDER_EPS)


def test_refusals(lib):
    """Each refusal of ctb_xchg_mul_mat's list returns -1 before anything reaches the GPU."""
    c, types, mats, attn, res0, norm_w, peers = _case("tiny-mixed-w2")
    parts = [[peers[k][r] for r in range(c[5])] for k in range(2 * X.N_LAYERS)]
    run = lambda base=0, ty=types, ps=parts, **over: X.run(lib, c, 1, ty, mats, attn, res0, norm_w, ps, base, **over)[0]
    assert run() == 0
    for over in ({"world": 1, "rank": 0}, {"world": 9, "rank": 0}, {"world": 2, "rank": 2}, {"world": 2, "rank": -1}, {"n_layers": 0}, {"steps": 0},
                 {"n_ff": 1000},                                  # n_ff off the 256-blocks: w2's K ranges too
                 {"n_ff": 256},                                   # more ranks than n_ff blocks
                 {"n_head_kv": 1},                                # a rank's 4 heads are half of an 8-head KV group
                 {"n_head": 5}):                                  # heads of 102.4: no shard
        assert run(**over) == -1, over
    for i, t in ((0, refs.Q8_0), (3, refs.Q4_0), (4, refs.F16)):
        ty = list(types)
        ty[i] = t
        assert run(ty=ty) == -1, (i, t)
    for k, r in ((0, 0), (3, 0)):
        ps = [list(p) for p in parts]
        ps[k][r] = None
        assert run(ps=ps) == -1, ("missing peer", k, r)
