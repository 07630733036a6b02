"""CPU checks of the fixtures of tests/test_tp_exchange_gpu.py (the tensor-sharded mode's fused exchange on one GPU): the planted
norm rows survive the split into rank partials, the expected values tell the right summation from the two likely mistakes,
and the shards the tests cut are the engine's."""
import ctypes as C

import numpy as np
import pytest

import refs
import tp_exchange_refs as X


@pytest.mark.parametrize("world", range(2, 9))
@pytest.mark.parametrize("k", [1024, 4096, 8192])
def test_planted_rows_split_into_rank_partials_sum_back_bit_for_bit(world, k):
    """The planted RMSNorm rows (refs.norm_order_rows), split by significand bit ranges into `world` partials, come back bit for
    bit from the fp32 rank-order sum the consumer forms; every rank holds non-zero parts, and no rank's part is the row."""
    rows, _, _ = refs.norm_order_rows(1, k, seed=k + world)
    for x in rows:
        parts = X.split_mantissa(x, world)
        assert np.array_equal(X.rank_sum(parts).view(np.uint32), x.view(np.uint32))
        for p in parts:
            assert np.count_nonzero(p) > 0 and not np.array_equal(p, x)


def test_split_mantissa_keeps_signs_zeros_and_subnormals():
    x = np.array([0.0, -0.0, 1.0, -3.75, np.float32(1e-40), -np.float32(1e-40), np.finfo(np.float32).max, -np.finfo(np.float32).tiny], np.float32)
    for world in range(2, 9):
        assert np.array_equal(X.rank_sum(X.split_mantissa(x, world)).view(np.uint32), x.view(np.uint32))


@pytest.mark.parametrize("case", list(X.CASES))
def test_expected_values_tell_the_rank_order_and_the_residual_rank(case):
    """With the case's shapes, types, world and random peer partials, the first consumer's expected outputs (oracle
    orc_rms_norm_mul + orc_mul_mat) change in at least one element when the partials are summed in reverse rank order (W >= 3;
    two fp32 terms commute, so at W = 2 the order cannot show and the outputs must stay the same), and when a rank other than
    0 adds the residual too: the GPU test's comparison would catch either mistake.  (Random weights: which weights the GPU
    test uses does not bear on the order of the sum.)"""
    c = X.CASES[case]
    c = c[:8] + ("random",) + c[9:]
    types, mats = X.model(c, seed=11)
    attn, res0, norm_w, peers = X.inputs(c, seed=12)
    for me in (0, c[6][-1]):
        args = (c, me, types, mats, attn, res0, norm_w, peers)
        want = X.expected(*args, own_peers=False, n_consumers=1)
        # (a rank other than 0 that adds the residual changes its own partial; rank 0 adds it anyway)
        for mistake in ({"reverse": True},) + (({"res_everywhere": True},) if me else ()):
            got = X.expected(*args, own_peers=False, n_consumers=1, **mistake)
            same = np.array_equal(got["outs"][0].view(np.uint32), want["outs"][0].view(np.uint32))
            assert same == ("reverse" in mistake and c[5] == 2), (case, me, mistake)


@pytest.mark.parametrize("case", list(X.CASES))
def test_shards_are_the_engines(lib, case):
    """The shard ranges the tests slice the full matrices by (tp_plan) are the ones csrc/engine.cu tp_shard gives every rank
    (ctb_tp_shard); each rank's query heads cover whole KV groups and every rank has heads and n_ff blocks."""
    E, nh, nkv, F, V, W = X.CASES[case][:6]
    hd, per_kv = E // nh, nh // nkv
    for r in range(W):
        out6 = (C.c_int * 6)()
        assert lib.ctb_tp_shard(E, nh, nkv, F, r, W, out6) == 0
        s = X.shard(E, nh, nkv, F, W, r)
        assert s["q"] == (out6[0] * hd, out6[1] * hd) and s["g"] == (out6[2] * hd, out6[3] * hd) and s["f"] == (out6[4], out6[5])
        assert out6[1] > out6[0] and out6[5] > out6[4] and out6[0] % per_kv == 0 and out6[1] % per_kv == 0


def test_uneven_splits_of_the_three_rank_case():
    """The 7B case at W = 3: 16 head groups of 2 heads deal 6 / 5 / 5, 43 n_ff blocks 15 / 14 / 14."""
    E, nh, nkv, F = X.CASES["7b-q4km-w3"][:4]
    sh = [X.shard(E, nh, nkv, F, 3, r) for r in range(3)]
    assert [(s["q"][1] - s["q"][0]) // 256 for s in sh] == [6, 5, 5]
    assert [(s["f"][1] - s["f"][0]) // 256 for s in sh] == [15, 14, 14]
