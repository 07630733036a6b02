"""GPU parity tests, op level: every CUDA stage of the hot path, called through the C ABI with host buffers, against
the plain-C oracle (oracle/ggml_oracle.c) on the same seeded inputs.

Bar: BIT-EXACT everywhere.  The oracle reproduces the reference's AVX2 accumulation order and FMA placement (it is pinned
bit for bit against the compiled reference in tests/test_oracle.py), and the CUDA kernels reproduce the same order, so
quantizers, norms, RoPE, embedding rows, every quantized dot product and the attention block must match to the last bit."""
import ctypes as C
import functools

import numpy as np
import pytest

import q3k_refs
import q41_q51_refs
import refs
from conftest import ptr
from q3k_refs import Q3_K
from q41_q51_refs import Q4_1, Q5_1
from refs import F16, F32, Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0, Q8_K, row_bytes

pytestmark = pytest.mark.gpu



def _rand_weights(t, k, m, seed, sigma=0.02):
    from ctransformers_b200 import synth
    return np.ascontiguousarray(synth.random_blocks(t, k, m, sigma, np.random.default_rng(seed))).view(np.uint8)


def _act(rng, k, scale=1.0):
    x = rng.standard_normal(k).astype(np.float32) * scale
    x[rng.integers(0, k, 8)] *= 17.0
    return x


@pytest.mark.parametrize("k", [256, 4096, 11008])
def test_quantize_q8_K_bit_exact(lib, k):
    o = refs.oracle()
    rng = np.random.default_rng(k)
    for trial in range(6):
        x = _act(rng, k, [1e-4, 1.0, 300.0][trial % 3])
        if trial == 3:
            x[:256] = 0.0                      # all-zero block → d = 0
        if trial == 4:
            x[5], x[9] = -3.5, 3.5             # |max| tie: the FIRST one fixes the sign
            x[:256] = np.clip(x[:256], -3.5, 3.5)
        a = np.zeros(row_bytes(Q8_K, k), np.uint8)
        b = np.zeros_like(a)
        o.orc_quantize_row_q8_K(ptr(x), ptr(a), k)
        assert lib.ctb_quantize_row_q8_K(ptr(x), ptr(b), k) == 0
        assert np.array_equal(a, b), f"trial {trial}: {(a != b).sum()} differing bytes"


@pytest.mark.parametrize("k", [32, 4096, 4544])
def test_quantize_q8_0_bit_exact(lib, k):
    o = refs.oracle()
    rng = np.random.default_rng(k + 1)
    for trial in range(4):
        x = _act(rng, k, [1e-3, 1.0, 50.0, 1.0][trial])
        if trial == 3:
            x[:32] = 0.0
        a = np.zeros(row_bytes(Q8_0, k), np.uint8)
        b = np.zeros_like(a)
        o.orc_quantize_row_q8_0(ptr(x), ptr(a), k)
        assert lib.ctb_quantize_row_q8_0(ptr(x), ptr(b), k) == 0
        assert np.array_equal(a, b)


def _same_bits(got, want, what=""):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError(f"{what}{': ' if what else ''}{int(bad.sum())} of {bad.size} values differ, the first at {at} "
                             f"({got[at]!r} for {want[at]!r}); max |diff| {np.abs(got - want).max():.3e}")


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K, Q4_0, Q5_0, Q8_0])
@pytest.mark.parametrize("k,m", [(256, 3), (4096, 64), (11008, 33)])
def test_mul_mat_vs_oracle(lib, t, k, m):
    o = refs.oracle()
    rng = np.random.default_rng(t * 1000 + k)
    w = _rand_weights(t, k, m, seed=t + k)
    n = 2
    x = np.stack([_act(rng, k), _act(rng, k, 0.05)])
    want = np.zeros((n, m), np.float32)
    got = np.zeros((n, m), np.float32)
    assert o.orc_mul_mat(t, ptr(w), ptr(x), ptr(want), k, m, n) == 0
    assert lib.ctb_mul_mat(t, ptr(w), ptr(x), ptr(got), k, m, n) == 0
    _same_bits(got, want)


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
@pytest.mark.parametrize("k,m", [(4096, 4096 + 37), (4096, 22016), (11008, 4096), (2048, 1184 + 8), (256, 9000)])
def test_mul_mat_full_size_partitions(lib, t, k, m):
    """Bench-sized shapes: many row tiles per CTA, warp ranges that start and end in the middle of a row (fold state handed from
    warp to warp, parked terms), ranges longer and shorter than a row, a ragged last tile — all bit-exact with the oracle."""
    o = refs.oracle()
    rng = np.random.default_rng(t * 77 + k + m)
    w = _rand_weights(t, k, m, seed=t + k + m)
    x = _act(rng, k)[None, :]
    want = np.zeros((1, m), np.float32)
    got = np.zeros((1, m), np.float32)
    assert o.orc_mul_mat(t, ptr(w), ptr(x), ptr(want), k, m, 1) == 0
    assert lib.ctb_mul_mat(t, ptr(w), ptr(x), ptr(got), k, m, 1) == 0
    _same_bits(got, want)


@pytest.mark.parametrize("k", [512, 1000])
def test_mul_mat_f16_weights(lib, k):
    """F16 weights take ggml_vec_dot_f16 with the activation row rounded to f16 (ggml.c:1665-1675, 2392-2426)."""
    o = refs.oracle()
    m = 24
    rng = np.random.default_rng(k)
    w = (rng.standard_normal((m, k)) * 0.05).astype(np.float16)
    x = _act(rng, k)[None]
    got = np.zeros((1, m), np.float32)
    assert lib.ctb_mul_mat(F16, ptr(w), ptr(x), ptr(got), k, m, 1) == 0
    x16 = x[0].astype(np.float16)
    want = np.array([o.orc_vec_dot_f16(k, ptr(np.ascontiguousarray(w[i])), ptr(x16)) for i in range(m)], np.float32)
    _same_bits(got[0], want)


def test_mul_mat_f32_weights(lib):
    k, m = 512, 16
    rng = np.random.default_rng(3)
    w = (rng.standard_normal((m, k)) * 0.05).astype(np.float32)
    x = _act(rng, k)[None]
    got = np.zeros((1, m), np.float32)
    assert lib.ctb_mul_mat(F32, ptr(w), ptr(x), ptr(got), k, m, 1) == 0
    assert np.allclose(got[0], w @ x[0], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("mode", [1, 2])
def test_norm_bit_exact(lib, mode):
    o = refs.oracle()
    n = 4096
    rng = np.random.default_rng(mode)
    x, w, b = _act(rng, n, 3.0), (1 + 0.1 * rng.standard_normal(n)).astype(np.float32), (0.1 * rng.standard_normal(n)).astype(np.float32)
    want, got = np.zeros(n, np.float32), np.zeros(n, np.float32)
    if mode == 1:
        o.orc_rms_norm_mul(ptr(x), ptr(w), ptr(want), n, 1e-5)
        assert lib.ctb_norm(1, ptr(x), ptr(w), None, ptr(got), n, 1e-5) == 0
    else:
        o.orc_layer_norm_mul_add(ptr(x), ptr(w), ptr(b), ptr(want), n, 1e-5)
        assert lib.ctb_norm(2, ptr(x), ptr(w), ptr(b), ptr(got), n, 1e-5) == 0
    assert np.array_equal(want.view(np.uint32), got.view(np.uint32)), f"{(want != got).sum()} of {n} differ, max {np.abs(want - got).max()}"


@pytest.mark.parametrize("mode,hd", [(0, 128), (2, 64), (0, 64)])
def test_rope_bit_exact(lib, mode, hd):
    o = refs.oracle()
    rng = np.random.default_rng(hd + mode)
    for pos in (0, 1, 37, 511):
        x = rng.standard_normal((8, hd)).astype(np.float32)
        want, got = x.copy(), x.copy()
        o.orc_rope(ptr(want), 8, hd, pos, mode, 10000.0, 1.0)
        assert lib.ctb_rope(ptr(got), 8, hd, pos, mode, 10000.0, 1.0) == 0
        assert np.array_equal(want.view(np.uint32), got.view(np.uint32)), f"pos {pos}: max diff {np.abs(want - got).max()}"


@pytest.mark.parametrize("n_head,n_kv,hd,T,n_total", [(4, 4, 128, 1, 1), (4, 4, 128, 300, 300), (8, 1, 64, 77, 77), (8, 2, 128, 512, 512),
                                                      (4, 4, 64, 21, 24), (4, 2, 128, 40, 64), (2, 2, 128, 33, 33), (2, 1, 64, 257, 300),
                                                      (4, 4, 128, 1500, 1500), (4, 1, 64, 2047, 2048), (2, 2, 128, 1027, 1027)])
def test_attention_bit_exact(lib, n_head, n_kv, hd, T, n_total):
    """n_total = row length of the reference's V·P mat-mul (n_past + N of the eval call): it fixes where the f16 dot switches
    from its 32 SIMD lanes to the scalar double tail, so it is part of the contract."""
    o = refs.oracle()
    rng = np.random.default_rng(T + hd)
    q = rng.standard_normal((n_head, hd)).astype(np.float32)
    kc = (rng.standard_normal((T, n_kv, hd)) * 0.7).astype(np.float16)          # [T][n_kv*hd]
    vt = rng.standard_normal((n_kv * hd, T)).astype(np.float16)                  # transposed, like the reference cache
    scale = np.float32(1.0 / np.sqrt(np.float32(hd)))
    got = np.zeros((n_head, hd), np.float32)
    assert lib.ctb_attention(ptr(q), ptr(kc), ptr(vt), ptr(got), n_head, n_kv, hd, T, n_total, float(scale)) == 0
    want = np.zeros((n_head, hd), np.float32)
    # the oracle's V·P dot runs over n_total entries: pad the transposed cache with zeros probabilities beyond T
    vpad = np.zeros((n_kv * hd, n_total), np.float16)
    vpad[:, :T] = vt
    for h in range(n_head):
        kvh = h // (n_head // n_kv)
        kslice = np.ascontiguousarray(kc[:, kvh, :])
        vslice = np.ascontiguousarray(vpad[kvh * hd:(kvh + 1) * hd])
        o.orc_attn_head_n(ptr(q[h]), ptr(kslice), hd, ptr(vslice), n_total, hd, T, n_total, float(scale), ptr(want[h]))
    _same_bits(got, want)


# ---- every attention implementation of the engine (ctb_attention_path), RoPE and the KV-cache store included
ATTN_PATHS = {0: "k_attn", 1: "step_ring", 2: "step_global", 3: "prefill"}
# (n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, rope mode, hard).  The call evaluates n_tok tokens at positions pos0..;
# chunk: they form one eval chunk, n_total = pos0 + n_tok + extra for all of them; else each is a chunk of its own with
# n_total = position + 1 + extra.  hard: scores over a wide range (most exp-table entries flush to 0) and all-zero V channels.
ATTN_CASES = {
    # T (= position + 1) across the edges of the step kernel's ring geometry: V chunks of 256 positions (nchv), channels per V
    # item (cv 8 -> 6 -> 4 -> 3 -> 2 at T 513 / 769 / 1025 / 1537), K items of 36 rows (hd 128), V items that fill a slot (T 2304)
    "T1-2": (8, 2, 128, 2304, 0, 2, False, 0, 0, False),
    "T31-33": (8, 2, 128, 2304, 30, 3, False, 0, 0, False),
    "T36-37": (8, 2, 128, 2304, 35, 2, False, 0, 0, False),
    "T255-257": (8, 2, 128, 2304, 254, 3, False, 0, 0, False),
    "T512-513": (8, 2, 128, 2304, 511, 2, False, 0, 0, False),
    "T768-769": (8, 2, 128, 2304, 767, 2, False, 0, 0, False),
    "T1024-1025": (8, 2, 128, 2304, 1023, 2, False, 0, 0, False),
    "T1536-1537": (8, 2, 128, 2304, 1535, 2, False, 0, 0, False),
    "T2047-2048": (8, 2, 128, 2304, 2046, 2, False, 0, 0, False),
    "T2304-full": (8, 2, 128, 2304, 2303, 1, False, 0, 0, False),
    # hd 64, MQA, neox: K items of 72 rows, a batch straddling a 256-position chunk, a full 32-token batch that fills the context
    "mqa-T72-73": (8, 1, 64, 2304, 71, 2, False, 0, 2, False),
    "mqa-straddle256": (8, 1, 64, 2304, 254, 5, True, 0, 2, False),
    "mqa-T513": (8, 1, 64, 2304, 512, 1, False, 0, 2, False),
    "mqa-T769": (8, 1, 64, 2304, 768, 1, False, 0, 2, False),
    "mqa-T1025": (8, 1, 64, 2304, 1024, 1, False, 0, 2, False),
    "mqa-T1537": (8, 1, 64, 2304, 1536, 1, False, 0, 2, False),
    "mqa-batch32-full": (8, 1, 64, 2304, 2272, 32, True, 0, 2, False),
    # more (head, channel group) tasks than SMs: Falcon-7B heads (71 x 2 = 142 tasks), 40 heads of 128 (160 tasks)
    "falcon7b-heads": (71, 1, 64, 2304, 1100, 5, True, 0, 2, False),
    "falcon7b-heads-ctx2000": (71, 1, 64, 2000, 300, 1, False, 0, 2, False),
    "40x128": (40, 40, 128, 1100, 1040, 3, False, 0, 0, False),
    # n_total > T: the V·P dot's split between SIMD lanes and the scalar tail; n_ctx not a multiple of 256
    "ntotal-tail": (4, 4, 128, 1000, 39, 1, False, 20, 0, False),
    "ntotal-lanes": (4, 4, 128, 1000, 39, 1, False, 30, 0, False),
    "ntotal-chunk": (16, 2, 64, 2304, 700, 5, True, 57, 0, False),
    "gqa8-batch32-ctx777": (16, 2, 64, 777, 600, 32, True, 0, 0, False),
    "batch1": (4, 4, 128, 600, 299, 1, True, 0, 0, False),
    # hard inputs
    "hard-hd128": (8, 2, 128, 1500, 1200, 3, True, 0, 0, True),
    "hard-hd64": (8, 1, 64, 600, 300, 5, True, 0, 2, True),
    # past the ring's reach (n_ctx > 2304) and past the batched kernel's scratch (n_ctx 4096)
    "ctx2305": (8, 2, 128, 2305, 2000, 2, False, 0, 0, False),
    "ctx3072": (8, 1, 64, 3072, 2900, 3, True, 0, 2, False),
    "ctx4096": (8, 1, 64, 4096, 4000, 2, True, 0, 2, False),
}


def _attn_inputs(n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, mode, hard):
    rng = np.random.default_rng(n_head * 7919 + hd * 31 + n_ctx + pos0 * 3 + n_tok)
    q = rng.standard_normal((n_tok, n_head * hd)).astype(np.float32) * (40.0 if hard else 1.0)
    k = (rng.standard_normal((n_tok, n_kv * hd)) * 0.7).astype(np.float32)
    v = rng.standard_normal((n_tok, n_kv * hd)).astype(np.float32)
    kc = (rng.standard_normal((n_ctx, n_kv * hd)) * 0.7).astype(np.float16).view(np.uint16)
    vc = rng.standard_normal((n_kv * hd, n_ctx)).astype(np.float16).view(np.uint16)
    if hard:   # a whole channel group of V and a few more channels are zero
        zero = list(range(32)) + [40, 77 % hd]
        vc[zero] = 0
        v[:, zero] = 0.0
    pos = pos0 + np.arange(n_tok)
    n_total = (np.full(n_tok, pos0 + n_tok + extra) if chunk else pos + 1 + extra).astype(np.int32)
    return q, k, v, kc, vc, n_total


@functools.lru_cache(maxsize=None)
def _attn_expected(case):
    n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, mode, hard = ATTN_CASES[case]
    q, k, v, kc, vc, n_total = _attn_inputs(*ATTN_CASES[case])
    return refs.attention_expected(q, k, v, kc, vc, n_head, n_kv, hd, pos0, n_total, mode, 10000.0, np.float32(1.0 / np.sqrt(np.float32(hd))))


@pytest.mark.parametrize("case", list(ATTN_CASES))
@pytest.mark.parametrize("path", list(ATTN_PATHS), ids=list(ATTN_PATHS.values()))
def test_attention_paths_bit_exact(lib, case, path):
    """Each attention implementation, launched as the engine launches it, on n_tok new tokens against the reference's attention
    block restated from oracle pieces: output, K cache and V cache identical to the last bit.  A path that cannot take the
    shape (the ring past 2304 positions, the batched kernel past its scratch or beyond 32 tokens) must refuse it."""
    n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, mode, hard = ATTN_CASES[case]
    q, k, v, kc, vc, n_total = _attn_inputs(*ATTN_CASES[case])
    out = np.zeros((n_tok, n_head * hd), np.float32)
    scale = np.float32(1.0 / np.sqrt(np.float32(hd)))
    rc = lib.ctb_attention_path(path, ptr(q), ptr(k), ptr(v), ptr(kc), ptr(vc), ptr(out), n_head, n_kv, hd, n_ctx, pos0, n_tok, ptr(n_total),
                                mode, 10000.0, float(scale))
    refused = (path == 1 and n_ctx > 2304) or (path == 3 and (n_ctx >= 4096 or n_tok > 32))
    if refused:
        assert rc == -1, "the path must refuse this shape"
        return
    assert rc == 0
    want, want_kc, want_vc = _attn_expected(case)
    _same_bits(out, want)
    assert np.array_equal(kc, want_kc), f"K cache: {int((kc != want_kc).sum())} entries differ"
    assert np.array_equal(vc, want_vc), f"V cache: {int((vc != want_vc).sum())} entries differ"


def test_attention_path_rejects_n_total_outside_the_context(lib):
    """n_total outside [position + 1, n_ctx] is refused, not run."""
    n_head, n_kv, hd, n_ctx, pos0, n_tok, *_ = ATTN_CASES["batch1"]
    q, k, v, kc, vc, _ = _attn_inputs(*ATTN_CASES["batch1"])
    out = np.zeros((n_tok, n_head * hd), np.float32)
    for bad in (pos0, n_ctx + 1):
        nt = np.array([bad], np.int32)
        assert lib.ctb_attention_path(2, ptr(q), ptr(k), ptr(v), ptr(kc), ptr(vc), ptr(out), n_head, n_kv, hd, n_ctx, pos0, n_tok, ptr(nt), 0,
                                      10000.0, 0.125) == -1


@pytest.mark.parametrize("t,src", [pytest.param(t, "random", id=str(t)) for t in (Q4_K, Q5_K, Q4_0, Q5_0)] +
                         [pytest.param(t, "edge", id=f"{t}-edge") for t in (Q4_K, Q5_K)])
def test_ffn_gate_vs_oracle(lib, t, src):
    """src "edge": refs.edge_blocks, every scale and min value and the quant extremes."""
    o = refs.oracle()
    k, m = 4096, 96
    rng = np.random.default_rng(t)
    gen = _rand_weights if src == "random" else refs.edge_blocks
    w1, w3 = gen(t, k, m, 1), gen(t, k, m, 2)
    x = _act(rng, k)
    g, u = np.zeros(m, np.float32), np.zeros(m, np.float32)
    o.orc_mul_mat(t, ptr(w1), ptr(x), ptr(g), k, m, 1)
    o.orc_mul_mat(t, ptr(w3), ptr(x), ptr(u), k, m, 1)
    s = np.zeros(m, np.float32)
    o.orc_silu(ptr(g), ptr(s), m)
    want = s * u
    got = np.zeros(m, np.float32)
    assert lib.ctb_ffn_gate(t, ptr(w1), ptr(w3), ptr(x), ptr(got), k, m) == 0
    _same_bits(got, want)


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K, Q4_0, Q5_0, Q8_0, F16, F32])
def test_get_row_bit_exact(lib, t):
    o = refs.oracle()
    k, rows = 512, 9
    if t == F32:
        tab = np.random.default_rng(1).standard_normal((rows, k)).astype(np.float32)
        want = tab
    elif t == F16:
        tab = np.random.default_rng(1).standard_normal((rows, k)).astype(np.float16)
        want = tab.astype(np.float32)
    else:
        tab = _rand_weights(t, k, rows, 5, sigma=1.0)
        want = np.zeros((rows, k), np.float32)
        getattr(o, "orc_dequantize_row_" + refs.TYPE_NAME[t])(ptr(tab), ptr(want), rows * k)
    for r in (0, 4, rows - 1):
        got = np.zeros(k, np.float32)
        assert lib.ctb_get_row(t, ptr(tab), k, rows, r, ptr(got)) == 0
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want[r]).view(np.uint32))


@pytest.mark.parametrize("t,src", [pytest.param(t, "refq", id=str(t)) for t in (Q4_K, Q5_K, Q6_K, Q4_0, Q5_0, Q8_0)] +
                         [pytest.param(t, "edge", id=f"{t}-edge") for t in (Q4_K, Q5_K, Q6_K)])
@pytest.mark.parametrize("k", [512, 1024, 2816])
def test_mul_mat_real_quantized_weights(lib, t, src, k):
    """src "refq": weights produced by the reference's quantizer (scale / min bit patterns the random-block generator does not
    write); "edge": refs.edge_blocks, every scale and min value (the pool's 6-bit scales stop at 26), all-zero and all-set quants,
    negative and subnormal d / dmin."""
    o = refs.oracle()
    rng = np.random.default_rng(k + t)
    m = 48
    w = (refs.reference_quantized_blocks if src == "refq" else refs.edge_blocks)(t, k, m, seed=k + t)
    x = _act(rng, k)[None]
    want, got = np.zeros((1, m), np.float32), np.zeros((1, m), np.float32)
    assert o.orc_mul_mat(t, ptr(w), ptr(x), ptr(want), k, m, 1) == 0
    assert lib.ctb_mul_mat(t, ptr(w), ptr(x), ptr(got), k, m, 1) == 0
    _same_bits(got, want)


# ---- the batched prefill kernel's mat-mul (csrc/prefill.cuh k_pstep, QUANT + GEMM phases) through ctb_prefill_mul_mat.  Its
# integer part is a second implementation of the K-quant dot products (scale digits on tensor cores), with its own mins chains,
# short-batch bookkeeping and epilogue; the expected values are orc_mul_mat with N = n_tok columns, prologue and epilogue from
# oracle pieces in the reference's order.
STORE, ADD, GELU, ADD2, SILU = 0, 1, 2, 3, 4
PF_SOURCES = {"random": _rand_weights, "refq": refs.reference_quantized_blocks, "edge": refs.edge_blocks}
PF_TOKENS = [1, 2, 7, 8, 9, 31, 32, 70]   # 70: launches of 32 + 32 + 6 on the same buffers, the short one after full ones
# name: (segments [(type, rows, epilogue)], K, n_tok, norm mode, x2 (x_mode 1), weight source)
PF_SHAPES = {
    "k256-m5": ([(Q5_K, 5, STORE)], 256, 70, 1, False, "edge"),
    "k256-m1": ([(Q6_K, 1, STORE)], 256, 9, 0, False, "edge"),            # one tile in the whole grid: one CTA, one team idle
    "k11008-m3-add": ([(Q4_K, 3, ADD)], 11008, 33, 0, False, "refq"),
    "3seg-mixed-epilogues": ([(Q4_K, 17, GELU), (Q5_K, 40, SILU), (Q6_K, 9, ADD2)], 1024, 40, 2, False, "edge"),
    "x2-add": ([(Q5_K, 50, ADD)], 2816, 12, 0, True, "edge"),
    # the bench's Llama-2-7B Q4_K_M layer (QKV with the more-bits V in Q6_K; gate + up; down on silu(gate) * up)
    "7b-qkv": ([(Q4_K, 4096, STORE), (Q4_K, 1024, STORE), (Q6_K, 1024, STORE)], 4096, 5, 1, False, "random"),
    "7b-gate-up": ([(Q4_K, 11008, SILU), (Q4_K, 11008, STORE)], 4096, 5, 1, False, "random"),
    "7b-down": ([(Q6_K, 4096, ADD)], 11008, 5, 0, True, "random"),
    # the Falcon-7B-shaped Q5_K_M layer: LayerNorm + fused wqkv and up (GELU), down + attention output + layer input
    "falcon7b-qkv-up": ([(Q5_K, 4736, STORE), (Q5_K, 18432, GELU)], 4608, 3, 2, False, "random"),
    "falcon7b-down": ([(Q6_K, 4608, ADD2)], 18432, 3, 0, False, "random"),
    # the output heads: the 7B's (RMSNorm, the embeddings written beside the logits) and the Falcon-7B-shaped one (LayerNorm)
    "7b-head": ([(Q6_K, 32000, STORE)], 4096, 3, 1, False, "random"),
    "falcon7b-head": ([(Q6_K, 65024, STORE)], 4608, 3, 2, False, "random"),
}


def _weights(t, k, m, seed, src):
    """m rows of k type-t weights from source src (PF_SOURCES); Q3_K, Q4_1 and Q5_1 from their checkers' own block makers."""
    if t == Q3_K:
        return q3k_refs.blocks(src, k, m, seed)
    if t in (Q4_1, Q5_1):
        Q = q41_q51_refs
        return {"random": Q.random_blocks, "refq": Q.reference_quantized_blocks, "edge": Q.edge_blocks}[src](t, k, m, seed)
    return np.ascontiguousarray(PF_SOURCES[src](t, k, m, seed))


def _pf_inputs(segs, k, n_tok, norm, with_x2, src, seed):
    rng = np.random.default_rng(seed)
    ws = [_weights(t, k, m, seed + 10 * i, src) for i, (t, m, _) in enumerate(segs)]
    x = np.stack([_act(rng, k, [1e-3, 1.0, 300.0][i % 3]) for i in range(n_tok)])
    x[0, :256] = 0.0                                                  # an all-zero block: Q8_K d = 0
    x2 = np.stack([_act(rng, k, 0.5) for _ in range(n_tok)]) if with_x2 else None
    nw = (1 + 0.1 * rng.standard_normal(k)).astype(np.float32)
    nb = (0.1 * rng.standard_normal(k)).astype(np.float32)
    W = sum(m for _, m, _ in segs)
    res = (rng.standard_normal((n_tok, W)) * 2).astype(np.float32)
    res2 = (rng.standard_normal((n_tok, W)) * 2).astype(np.float32)
    return ws, x, x2, nw, nb, res, res2


def _oracle_mul_mat(t, w, y, k, m):
    """[n_tok][m]: ggml_mul_mat of m rows of type-t weights by the rows y, each quantized to the type's activation format; F16
    weights take ggml_vec_dot_f16 on y rounded to f16, as in test_mul_mat_f16_weights."""
    n_tok = y.shape[0]
    if t == F16:
        o = refs.oracle()
        w16, y16 = w.view(np.float16).reshape(m, k), y.astype(np.float16)
        return np.array([[o.orc_vec_dot_f16(k, ptr(w16[j]), ptr(y16[i])) for j in range(m)] for i in range(n_tok)], np.float32)
    v = np.zeros((n_tok, m), np.float32)
    assert refs.oracle().orc_mul_mat(t, ptr(w), ptr(y), ptr(v), k, m, n_tok) == 0
    return v


def _pf_expected(segs, ws, k, x, x2, norm, nw, nb, res, res2, eps=1e-5):
    """(out, y): y = the rows the mat-muls take (the normalised rows, x * x2, or x), out = every segment's mat-mul of y with its
    epilogue, side by side."""
    o = refs.oracle()
    n_tok = x.shape[0]
    y = np.zeros_like(x)
    for i in range(n_tok):
        if norm == 1:
            o.orc_rms_norm_mul(ptr(x[i]), ptr(nw), ptr(y[i]), k, eps)
        elif norm == 2:
            o.orc_layer_norm_mul_add(ptr(x[i]), ptr(nw), ptr(nb), ptr(y[i]), k, eps)
        else:
            y[i] = x[i] if x2 is None else x[i] * x2[i]
    outs, off = [], 0
    for (t, m, epi), w in zip(segs, ws):
        v = _oracle_mul_mat(t, w, y, k, m)
        if epi == ADD:
            v = v + res[:, off:off + m]
        elif epi == ADD2:
            v = (v + res[:, off:off + m]) + res2[:, off:off + m]
        elif epi in (GELU, SILU):
            a = np.zeros_like(v)
            (o.orc_gelu if epi == GELU else o.orc_silu)(ptr(v), ptr(a), v.size)
            v = a
        outs.append(v)
        off += m
    return np.concatenate(outs, axis=1), y


def _pf_run(lib, segs, ws, k, x, x2, norm, nw, nb, res, res2, n_ctx=512, hd=128, eps=1e-5):
    """ctb_prefill_mul_mat on the first n_tok rows; returns (rc, out, ring slots)."""
    n_tok = x.shape[0]
    nseg = len(segs)
    types, rows, epi = (np.array([s[j] for s in segs], np.int32) for j in range(3))
    wp = (C.c_void_p * max(nseg, 1))(*[w.ctypes.data for w in ws])
    out = np.full((n_tok, int(rows.sum())), np.nan, np.float32)
    slots = np.zeros(1, np.int32)
    rc = lib.ctb_prefill_mul_mat(nseg, ptr(types), C.cast(wp, C.c_void_p), ptr(rows), k, n_tok, ptr(x), None if x2 is None else ptr(x2),
                                 norm, ptr(nw), ptr(nb), eps, ptr(epi), ptr(res), ptr(res2), ptr(out), n_ctx, hd, ptr(slots))
    return rc, out, int(slots[0])


@functools.lru_cache(maxsize=None)
def _pf_case(t, src):
    segs = [(t, 37, STORE)]
    ws, x, x2, nw, nb, res, res2 = _pf_inputs(segs, 11008, max(PF_TOKENS), 0, False, src, seed=t)
    return segs, ws, x, res, res2, nw, nb, _pf_expected(segs, ws, 11008, x, None, 0, nw, nb, res, res2)[0]


@pytest.mark.parametrize("src", list(PF_SOURCES))
@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
def test_prefill_mul_mat_types_and_weight_sources(lib, t, src):
    """Every K-quant type on random blocks, the reference's quantizer's blocks and the edge blocks (every scale and min, quant
    extremes, negative and subnormal d / dmin); K = 11008 (43 blocks: a ragged last work item for every chunk size 4 / 3 / 2),
    M = 37 (a partial last tile), and 1 .. 70 tokens: partial token groups, one full launch, and a short launch after full ones.
    Token i is the same row in every run, so each run is checked against the first rows of one 70-column oracle mat-mul."""
    segs, ws, x, res, res2, nw, nb, want = _pf_case(t, src)
    for n in PF_TOKENS:
        rc, got, _ = _pf_run(lib, segs, ws, 11008, x[:n], None, 0, nw, nb, res[:n], res2[:n])
        assert rc == 0
        _same_bits(got, want[:n], f"n_tok {n}")


@functools.lru_cache(maxsize=None)
def _pf_shape_expected(case):
    segs, k, n_tok, norm, with_x2, src = PF_SHAPES[case]
    ws, x, x2, nw, nb, res, res2 = _pf_inputs(segs, k, n_tok, norm, with_x2, src, seed=len(case) * 131 + k)
    return (ws, x, x2, nw, nb, res, res2), _pf_expected(segs, ws, k, x, x2, norm, nw, nb, res, res2)


@pytest.mark.parametrize("case,kernel", [pytest.param(c, "prefill", id=c) for c in PF_SHAPES] +
                         [pytest.param(c, "decode", id=f"decode-{c}") for c in PF_SHAPES])
def test_prefill_mul_mat_shapes(lib, monkeypatch, case, kernel):
    """Rows below one tile, single-tile grids, several segments of different types and epilogues in one phase, x_mode 1, RMSNorm
    and LayerNorm prologues, the 7B-shaped projections the prefill2048 bench runs and the output heads: bit-exact with the
    oracle, through the batched prefill kernel and through the decode step's mat-vec phase in both its launch shapes (there
    the phase's input, as norm_out, too)."""
    segs, k, n_tok, norm, with_x2, src = PF_SHAPES[case]
    (ws, x, x2, nw, nb, res, res2), (want, y) = _pf_shape_expected(case)
    if kernel == "decode":
        for paired in _launch_shapes(monkeypatch):
            _dec_check(lib, segs, ws, k, (x, x2, norm, nw, nb, res, res2), (want, y), _dec_launch(paired, k), f"paired {paired}")
        return
    rc, got, _ = _pf_run(lib, segs, ws, k, x, x2, norm, nw, nb, res, res2)
    assert rc == 0
    _same_bits(got, want)


def _pf_accepts(lib, n_ctx, hd):
    w = refs.edge_blocks(Q4_K, 256, 1, 0)
    x = np.ones((1, 256), np.float32)
    z = np.zeros((1, 1), np.float32)
    return _pf_run(lib, [(Q4_K, 1, STORE)], [w], 256, x, None, 0, x[0], x[0], z, z, n_ctx=n_ctx, hd=hd)


def test_prefill_mul_mat_deepest_and_shallowest_ring(lib):
    """The ring depth follows n_ctx: the batched kernel's attention scratch shares shared memory with it.  The same mat-mul at the
    deepest ring (a short context) and at the shallowest one an engine can pick (the longest context that still gets batched
    prefill: 2 slots per team, so every slot's phase parity flips on every other item), one context longer being refused."""
    hd = 64
    lo, hi = 64, 8192
    assert _pf_accepts(lib, lo, hd)[0] == 0 and _pf_accepts(lib, hi, hd)[0] == -1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _pf_accepts(lib, mid, hd)[0] == 0:
            lo = mid
        else:
            hi = mid
    segs = [(Q6_K, 40, STORE), (Q5_K, 24, ADD), (Q4_K, 20, SILU)]
    ws, x, x2, nw, nb, res, res2 = _pf_inputs(segs, 11008, 70, 1, False, "edge", seed=5)
    want, _ = _pf_expected(segs, ws, 11008, x, None, 1, nw, nb, res, res2)
    depths = {}
    for n_ctx in (16, lo):
        rc, got, depths[n_ctx] = _pf_run(lib, segs, ws, 11008, x, None, 1, nw, nb, res, res2, n_ctx=n_ctx, hd=hd)
        assert rc == 0
        _same_bits(got, want)
    assert depths[lo] == 4 and depths[16] > depths[lo], depths


def test_prefill_mul_mat_refuses_what_the_kernel_cannot_take(lib):
    w = refs.edge_blocks(Q4_K, 512, 16, 0)
    x = np.ones((2, 512), np.float32)
    r = np.zeros((2, 64), np.float32)
    ok = _pf_run(lib, [(Q4_K, 16, STORE)], [w], 512, x, None, 0, x[0], x[0], r, r)
    assert ok[0] == 0
    assert _pf_run(lib, [(Q8_0, 16, STORE)], [_rand_weights(Q8_0, 512, 16, 0)], 512, x, None, 0, x[0], x[0], r, r)[0] == -1
    x384 = np.ones((2, 384), np.float32)
    assert lib.ctb_prefill_mul_mat(1, ptr(np.array([Q4_K], np.int32)), C.cast((C.c_void_p * 1)(w.ctypes.data), C.c_void_p),
                                   ptr(np.array([16], np.int32)), 384, 2, ptr(x384), None, 0, None, None, 1e-5, ptr(np.zeros(1, np.int32)),
                                   None, None, ptr(r), 512, 128, None) == -1
    assert _pf_run(lib, [(Q4_K, 4, STORE)] * 4, [w] * 4, 512, x, None, 0, x[0], x[0], r, r)[0] == -1
    assert _pf_run(lib, [(Q4_K, 16, STORE)], [w], 512, x[:0], None, 0, x[0], x[0], r, r)[0] == -1


# ---- the decode step's mat-vec phase through ctb_decode_mul_mat: routed as the engine routes it, K-quant matrices to the
# persistent step kernel (csrc/stream.cuh k_step), the other types to k_matvec, one launch per token.  The step kernel runs in
# clusters of two CTAs that split the input's norm, normalisation and Q8_K quantization (csrc/matvec.cuh stage_q8k_pair) unless
# CTB_ST_CLUSTER=0 or the input is wider than 80 Q8_K blocks; every test runs both launch shapes in one process and checks the
# launch it meant to test.  Expected values: _pf_expected, as for the batched prefill kernel.
DEC_PAIR_MAX_NB = 80                           # widest input a pair stages: 40 blocks per rank, two groups of 16 per thread
DEC_SEGS = [(Q4_K, 17, ADD), (Q6_K, 5, SILU), (Q5_K, 30, GELU)]
DEC_NORMS = {"none": (0, False), "rms": (1, False), "layer": (2, False), "x_mode1": (0, True)}   # name: (norm mode, x2)
NORM_KS = (256, 512, 1024, 4096, 4608, 8192, 11008)   # test_norm_order.KS that the step kernel takes


def _launch_shapes(monkeypatch):
    """Yields False with CTB_ST_CLUSTER=0, then True with pairs wanted (the default); step_pair_wanted reads the variable on
    every plan."""
    monkeypatch.setenv("CTB_ST_CLUSTER", "0")
    yield False
    monkeypatch.delenv("CTB_ST_CLUSTER")
    yield True


def _dec_launch(paired, k):
    """The {kernel, CTAs per cluster} a K-quant phase of width k must get: k_step, paired when pairs are wanted and k fits."""
    return 1, 2 if paired and k // 256 <= DEC_PAIR_MAX_NB else 1


def _pair_block0(nb, rank):
    """csrc/matvec.cuh pair_block0: the first Q8_K block rank 0 / 1 stages (rank 0 takes the odd block); 2 gives nb."""
    return (0, (nb + 1) // 2, nb)[rank]


def _dec_run(lib, segs, ws, k, x, x2, norm, nw, nb, res, res2, repeat=1, eps=1e-5):
    """ctb_decode_mul_mat on the rows of x; returns (rc, out, norm_out, (kernel, CTAs per cluster))."""
    n_tok, nseg = x.shape[0], len(segs)
    types, rows, epi = (np.array([s[j] for s in segs] or [0], np.int32) for j in range(3))
    wp = (C.c_void_p * max(nseg, 1))(*[w.ctypes.data for w in ws])
    out = np.full((n_tok, int(rows[:nseg].sum())), np.nan, np.float32)
    y = np.full((n_tok, k), np.nan, np.float32)
    launch = np.full(2, -1, np.int32)
    opt = lambda a: None if a is None else ptr(a)
    rc = lib.ctb_decode_mul_mat(nseg, ptr(types), C.cast(wp, C.c_void_p), ptr(rows), k, n_tok, ptr(x), opt(x2), norm, opt(nw), opt(nb), eps,
                                ptr(epi), opt(res), opt(res2), ptr(out), ptr(y), repeat, ptr(launch))
    return rc, out, y, tuple(int(v) for v in launch)


def _dec_check(lib, segs, ws, k, inputs, expected, launch, what, repeat=1, eps=1e-5):
    """One ctb_decode_mul_mat call: the launch it reports, out and norm_out against expected = (out, y) bit for bit."""
    rc, got, got_y, ran = _dec_run(lib, segs, ws, k, *inputs, repeat=repeat, eps=eps)
    assert rc == 0, what
    assert ran == launch, f"{what}: launched {ran}, meant {launch}"
    _same_bits(got, expected[0], f"{what}: out")
    _same_bits(got_y, expected[1], f"{what}: norm_out")


@functools.lru_cache(maxsize=None)
def _dec_inputs(nb):
    """_pf_inputs for DEC_SEGS at width 256·nb (tokens at scales 1e-3, 1 and 300, edge weights), with planted blocks: token 0 has
    block 0 and rank 1's first block all zero, token 1 the block a pair's rank 0 stages beyond rank 1's count (nb odd), and
    token 2 |max| ties in the first two blocks of each rank (one warp's two half-warps): in each block the largest |x| twice,
    with both signs, in two threads of the block, the first one negative in one block and positive in the next.  The norm
    weights are 1 at the tied elements, so that RMSNorm keeps the ties, and so is x2."""
    k = 256 * nb
    ws, x, x2, nw, nbias, res, res2 = _pf_inputs(DEC_SEGS, k, 3, 0, True, "edge", seed=7000 + nb)
    b1 = _pair_block0(nb, 1)
    if b1 < nb:
        x[0, 256 * b1:256 * (b1 + 1)] = 0.0
    if nb % 2:
        x[1, 256 * (b1 - 1):256 * b1] = 0.0
    big = np.float32(4 * np.abs(x[2]).max())
    for b in sorted({0, b1} - {nb}):
        for j, (first, second) in enumerate([(16 * 2 + 3, 16 * 9 + 1), (16 * 1 + 5, 16 * 14 + 2)][:min(2, nb - b)]):
            i0, i1 = 256 * (b + j) + first, 256 * (b + j) + second
            sign = np.float32(-1 if j == 0 else 1)
            x[2, i0], x[2, i1] = sign * big, -sign * big
            nw[[i0, i1]] = 1.0
            x2[2, [i0, i1]] = 1.0
    return ws, x, x2, nw, nbias, res, res2


def _dec_modes(nb):
    """(name, inputs, expected) of every DEC_NORMS mode on _dec_inputs(nb)."""
    ws, x, x2, nw, nbias, res, res2 = _dec_inputs(nb)
    for name, (norm, with_x2) in DEC_NORMS.items():
        inputs = (x, x2 if with_x2 else None, norm, nw, nbias, res, res2)
        yield name, inputs, _pf_expected(DEC_SEGS, ws, 256 * nb, *inputs)


@pytest.mark.parametrize("nb", list(range(1, DEC_PAIR_MAX_NB + 2)) + [112])
def test_decode_mul_mat_widths(lib, monkeypatch, nb):
    """Every input width the paired staging splits differently, K = 256·nb: nb odd (rank 0 stages the extra block), nb = 1 (rank
    1 stages nothing), nb >= 41 (a thread's second group of 16), nb = 80 (40 blocks per rank fill both groups), nb = 81 and the
    28672-wide down projection's 112 (unpaired).  Each width runs three segments of different types and epilogues without a
    norm, with RMSNorm, with LayerNorm and on x * x2 (x_mode 1); at the widths of NORM_KS also the rows whose fp64 norm sums
    round differently in another order (refs.norm_order_rows), so that the element-order fallback runs in the paired build."""
    k = 256 * nb
    ws = _dec_inputs(nb)[0]
    cases = list(_dec_modes(nb))
    if k in NORM_KS:
        for mode in (1, 2):
            rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
            z = np.zeros((rows.shape[0], sum(m for _, m, _ in DEC_SEGS)), np.float32)
            inputs = (rows, None, mode, w, b, z, z)
            cases.append((f"planted {mode}", inputs, _pf_expected(DEC_SEGS, ws, k, *inputs, eps=refs.NORM_ORDER_EPS)))
    for paired in _launch_shapes(monkeypatch):
        for name, inputs, expected in cases:
            eps = refs.NORM_ORDER_EPS if name.startswith("planted") else 1e-5
            _dec_check(lib, DEC_SEGS, ws, k, inputs, expected, _dec_launch(paired, k), f"nb {nb}, {name}, paired {paired}", eps=eps)


def _dec_accepts(lib, nb):
    segs = [(t, 1, STORE) for t, _, _ in DEC_SEGS]
    ws = [refs.edge_blocks(t, 256 * nb, 1, 0) for t, _, _ in segs]
    x = np.ones((1, 256 * nb), np.float32)
    z = np.zeros((1, len(segs)), np.float32)
    return _dec_run(lib, segs, ws, 256 * nb, x, None, 0, None, None, z, z)[0] == 0


def test_decode_mul_mat_widest_input(lib, monkeypatch):
    """The widest input the step kernel's shared memory takes beside its ring (found by bisection, in each launch shape: the
    paired builds hold more static shared memory) runs every mode bit-exact, and one block wider is refused."""
    for paired in _launch_shapes(monkeypatch):
        lo, hi = 112, 1024
        assert _dec_accepts(lib, lo) and not _dec_accepts(lib, hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if _dec_accepts(lib, mid) else (lo, mid)
        for name, inputs, expected in _dec_modes(lo):
            _dec_check(lib, DEC_SEGS, _dec_inputs(lo)[0], 256 * lo, inputs, expected, (1, 1), f"nb {lo}, {name}, paired {paired}")


@pytest.mark.parametrize("nb", [43, 72])
def test_decode_mul_mat_exchange_rounds(lib, monkeypatch, nb):
    """A pair's exchange rounds alternate two mbarriers and two partial buffers, and a phase takes one round (no norm), two
    (RMSNorm) or three (LayerNorm): the same phase 1, 2 and 3 times in one launch reaches every parity sequence, and every
    repeat must give the oracle's bits."""
    ws = _dec_inputs(nb)[0]
    for paired in _launch_shapes(monkeypatch):
        for name, inputs, expected in _dec_modes(nb):
            for repeat in (1, 2, 3):
                _dec_check(lib, DEC_SEGS, ws, 256 * nb, inputs, expected, _dec_launch(paired, 256 * nb), f"{name}, repeat {repeat}, paired {paired}",
                           repeat=repeat)


def _pow2_scaled(t, w, m):
    """Edge blocks of type t with each row's d (and dmin) set to ±2^e, e cycling from -24 (the smallest f16 subnormal) to 15."""
    blk = w.reshape(-1, refs.BLOCK[t][1]).copy()
    rows = blk.reshape(m, -1, blk.shape[1])
    e = np.arange(m) % 40 - 24
    d = (np.exp2(e) * np.where(np.arange(m) % 3 == 1, -1, 1)).astype(np.float16).view(np.uint8).reshape(m, 1, 2)
    for at in ((208,) if t == Q6_K else (0, 2)):
        rows[:, :, at:at + 2] = d
    return np.ascontiguousarray(rows.reshape(-1))


def test_mul_mat_epilogue_fp16_range(lib, monkeypatch):
    """Row values across the whole fp16 range meet the SiLU / GELU tables (indexed by the value rounded to fp16): zeros,
    subnormals, normals and values past 65504 (the index is ±inf; SiLU(-inf) and GELU(-inf) are NaNs whose sign and payload
    the output keeps, as the reference's F16C conversion does); and the ADD / ADD2 residual sums with residuals that cancel
    the row value exactly.  Through the decode step's mat-vec phase in both launch shapes and the batched prefill."""
    k, m = 1024, 40
    base = [(Q4_K, m, STORE), (Q5_K, m, STORE), (Q6_K, m, STORE)]
    ws, x, _, nw, nbias, res, res2 = _pf_inputs(base, k, 3, 0, False, "edge", seed=99)
    ws = [_pow2_scaled(t, w, m) for (t, _, _), w in zip(base, ws)]
    x[0] *= np.float32(1e-3)
    v, _ = _pf_expected(base, ws, k, x, None, 0, nw, nbias, res, res2)
    a = np.abs(v)
    ranges = {"fp16 zero": a < 2.0 ** -25, "fp16 subnormal": (a >= 2.0 ** -25) & (a < 2.0 ** -14), "fp16 normal": (a >= 2.0 ** -14) & (a <= 65504),
              "fp16 inf": a >= 65520}
    assert all(r.any() for r in ranges.values()), {n: int(r.sum()) for n, r in ranges.items()}
    cancel = np.arange(3 * m) % 2 == 0
    res = np.where(cancel, -v, res).astype(np.float32)              # v + res: exactly 0
    res2 = np.where(cancel, np.float32(-0.0), res2).astype(np.float32)
    res2[:, 1::4] = -(v + res)[:, 1::4]                               # (v + res) + res2: exactly 0
    for segs in ([(Q4_K, m, SILU), (Q5_K, m, GELU), (Q6_K, m, ADD)], [(Q4_K, m, ADD2), (Q5_K, m, ADD), (Q6_K, m, ADD2)]):
        inputs = (x, None, 0, nw, nbias, res, res2)
        want, y = _pf_expected(segs, ws, k, *inputs)
        for paired in _launch_shapes(monkeypatch):
            _dec_check(lib, segs, ws, k, inputs, (want, y), _dec_launch(paired, k), f"{segs}, paired {paired}")
        rc, got, _ = _pf_run(lib, segs, ws, k, x, None, 0, nw, nbias, res, res2)
        assert rc == 0
        _same_bits(got, want, f"{segs}, prefill")


# name: (segments, K, weight source); the activation formats Q8_0 (Q4_0 / Q5_0 / Q8_0), Q8_1 (Q4_1 / Q5_1) and F16
DEC_LEGACY = {
    "q8_0-k4544": ([(Q4_0, 21, ADD), (Q5_0, 9, SILU), (Q8_0, 36, GELU)], 4544, "refq"),
    "q8_0-k11008": ([(Q8_0, 21, ADD2), (Q4_0, 9, GELU), (Q5_0, 36, SILU)], 11008, "refq"),
    "q8_1-k4544": ([(Q4_1, 21, ADD), (Q5_1, 9, SILU), (Q4_1, 36, GELU)], 4544, "edge"),
    "q8_1-k11008": ([(Q5_1, 21, ADD2), (Q4_1, 9, GELU), (Q5_1, 36, SILU)], 11008, "random"),
    "f16-k1000": ([(F16, 7, ADD2), (F16, 9, GELU)], 1000, "random"),
    "f16-k4544": ([(F16, 5, SILU), (F16, 12, ADD)], 4544, "random"),
}


@pytest.mark.parametrize("case", list(DEC_LEGACY))
def test_decode_mul_mat_legacy_types(lib, monkeypatch, case):
    """The weight types the step kernel does not take run through k_matvec with the same prologues, x_mode 1 and epilogues,
    at Falcon-7B's 4544 and Llama-7B's 11008 (neither a multiple of k_matvec's 8192 elements per pass)."""
    segs, k, src = DEC_LEGACY[case]
    ws, x, x2, nw, nbias, res, res2 = _pf_inputs(segs, k, 3, 0, True, src, seed=k + len(case))
    for name, (norm, with_x2) in DEC_NORMS.items():
        inputs = (x, x2 if with_x2 else None, norm, nw, nbias, res, res2)
        expected = _pf_expected(segs, ws, k, *inputs)
        for paired in _launch_shapes(monkeypatch):
            _dec_check(lib, segs, ws, k, inputs, expected, (0, 1), f"{name}, paired {paired}")


@pytest.mark.parametrize("k", [4096, 11008])
def test_decode_mul_mat_q3k_unpaired(lib, monkeypatch, k):
    """A phase with a Q3_K matrix (beside Q4_K and Q6_K ones, as in a Q3_K_M layer) runs k_step's Q3 build, never paired."""
    segs = [(Q3_K, 17, ADD), (Q4_K, 5, SILU), (Q6_K, 30, GELU)]
    ws, x, x2, nw, nbias, res, res2 = _pf_inputs(segs, k, 3, 0, True, "edge", seed=k + 3)
    for name, (norm, with_x2) in DEC_NORMS.items():
        inputs = (x, x2 if with_x2 else None, norm, nw, nbias, res, res2)
        expected = _pf_expected(segs, ws, k, *inputs)
        for paired in _launch_shapes(monkeypatch):
            _dec_check(lib, segs, ws, k, inputs, expected, (1, 1), f"{name}, paired {paired}")


def test_decode_mul_mat_refuses_what_the_engine_never_builds(lib):
    w = refs.edge_blocks(Q4_K, 512, 16, 0)
    x = np.ones((2, 512), np.float32)
    r = np.zeros((2, 64), np.float32)
    run = lambda segs, ws, k=512, x=x, x2=None, norm=0, res=r, res2=r, repeat=1: _dec_run(lib, segs, ws, k, x, x2, norm, x[0], x[0], res, res2,
                                                                                         repeat=repeat)[0]
    assert run([(Q4_K, 16, STORE)], [w]) == 0
    assert run([(Q4_K, 16, STORE), (Q8_0, 16, STORE)], [w, _rand_weights(Q8_0, 512, 16, 0)]) == -1     # Q8_K beside Q8_0 activations
    assert run([(Q4_K, 16, STORE)], [w], x2=x, norm=1) == -1
    assert run([(Q4_K, 16, ADD)], [w], res=None) == -1
    assert run([(Q4_K, 16, ADD2)], [w], res2=None) == -1
    assert run([(Q4_K, 16, STORE)], [w], k=384, x=np.ones((2, 384), np.float32)) == -1
    assert run([(Q4_0, 16, STORE)], [_rand_weights(Q4_0, 512, 16, 0)], k=48, x=np.ones((2, 48), np.float32)) == -1
    assert run([], []) == -1
    assert run([(Q4_K, 4, STORE)] * 4, [w] * 4) == -1
    assert run([(Q4_K, 16, STORE)], [w], repeat=0) == -1 and run([(Q4_K, 16, STORE)], [w], repeat=5) == -1
