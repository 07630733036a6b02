"""CPU tests that pin the oracle: the plain-C restatement (oracle/ggml_oracle.c) against (1) the committed golden
vectors that the unmodified reference produced (tests/golden/make_golden.py), (2) what the compiled reference itself
returned for further inputs (tests/golden/reference_runs.npz), (3) the known-answer thresholds of upstream test-quantize-fns.cpp
(models/submodules/llama.cpp/tests/test-quantize-fns.cpp:16-31, 76-113)."""
from pathlib import Path

import numpy as np
import pytest

import refs
from refs import Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0, Q8_K, ptr, row_bytes

GOLD = Path(__file__).resolve().parent / "golden"
TYPES = [(Q4_0, Q8_0), (Q5_0, Q8_0), (Q8_0, Q8_0), (Q4_K, Q8_K), (Q5_K, Q8_K), (Q6_K, Q8_K)]


@pytest.fixture(scope="module")
def kat():
    return np.load(GOLD / "kat_quant.npz")


def _oracle_quant(t, x):
    o = refs.oracle()
    out = np.zeros(row_bytes(t, x.size), np.uint8)
    (o.orc_quantize_row_q8_K if t == Q8_K else o.orc_quantize_row_q8_0)(ptr(np.ascontiguousarray(x)), ptr(out), x.size)
    return out


@pytest.mark.parametrize("k", [256, 1024])
def test_activation_quantizers_match_golden(kat, k):
    x = kat[f"x_{k}"]
    assert np.array_equal(_oracle_quant(Q8_K, x), kat[f"q8k_{k}"])
    assert np.array_equal(_oracle_quant(Q8_0, x), kat[f"q80_{k}"])


@pytest.mark.parametrize("t,at", TYPES)
def test_vec_dot_and_dequant_match_golden(kat, t, at):
    o = refs.oracle()
    wq, x = kat[f"wq_{t}"], kat["x_1024"]
    act = _oracle_quant(at, x)
    fn = getattr(o, f"orc_vec_dot_{refs.TYPE_NAME[t]}_{'q8_K' if at == Q8_K else 'q8_0'}")
    got = np.array([fn(1024, ptr(np.ascontiguousarray(wq[i])), ptr(act)) for i in range(wq.shape[0])], np.float32)
    want = kat[f"dot_{t}"]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "oracle dot must equal the reference bit for bit"
    deq = np.zeros_like(kat[f"deq_{t}"])
    getattr(o, "orc_dequantize_row_" + refs.TYPE_NAME[t])(ptr(np.ascontiguousarray(wq)), ptr(deq), deq.size)
    assert np.array_equal(deq.view(np.uint32), kat[f"deq_{t}"].view(np.uint32))


@pytest.mark.parametrize("t,at", TYPES)
def test_upstream_quantize_fns_thresholds(kat, t, at):
    """test-quantize-fns.cpp: dot(q(x), q8(y)) error / n < 0.02 on 0.1 + 2cos(i + offset), n = 4096·32 there, 4096 here;
    round-trip array_rmse (sqrt(sum sq)/n, test-quantize-fns.cpp:34-41) < 0.002.  Weights quantized by the reference (golden file) are not available for this vector, so the
    round trip uses the activation types we quantize ourselves, and the dot uses golden weights vs the float dot."""
    o = refs.oracle()
    wq, x, w = kat[f"wq_{t}"], kat["x_1024"], kat["w_f32"]
    act = _oracle_quant(at, x)
    fn = getattr(o, f"orc_vec_dot_{refs.TYPE_NAME[t]}_{'q8_K' if at == Q8_K else 'q8_0'}")
    for i in range(wq.shape[0]):
        got = fn(1024, ptr(np.ascontiguousarray(wq[i])), ptr(act))
        assert abs(got - float(w[i] @ x)) / 1024 < 0.02
    # Q8_0 / Q8_K round trip of the synthetic test vector
    n = 4096
    v = (0.1 + 2 * np.cos(np.arange(n) + 1.0)).astype(np.float32)
    q = _oracle_quant(Q8_0, v).reshape(-1, 34)
    d = q[:, :2].copy().view(np.float16).astype(np.float32)
    back = (q[:, 2:].view(np.int8).astype(np.float32) * d).reshape(-1)
    assert np.sqrt(np.sum((back - v) ** 2)) / n < 0.002   # upstream array_rmse = sqrt(sum of squares) / n


def test_fp16_conversions_exhaustive():
    o = refs.oracle()
    bits = np.arange(65536, dtype=np.uint16)
    f = bits.view(np.float16).astype(np.float32)
    mine = np.array([o.orc_fp16_to_fp32(int(b)) for b in bits], np.float32)
    ok = ~np.isnan(f)
    assert np.array_equal(mine.view(np.uint32)[ok], f.view(np.uint32)[ok])
    back = np.array([o.orc_fp32_to_fp16(float(v)) for v in f[ok]], np.uint16)
    assert np.array_equal(back, bits[ok])
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(20000) * rng.choice([1e-8, 1e-5, 1e-3, 1, 100, 7e4], 20000)).astype(np.float32)
    assert np.array_equal(np.array([o.orc_fp32_to_fp16(float(v)) for v in x], np.uint16), x.astype(np.float16).view(np.uint16))


def _decode_k_blocks(t, blocks):
    """(scales, mins, quants, d, dmin) of K-quant blocks, read from their bytes the way the reference's dequantizers read them
    (get_scale_min_k4, k_quants.c:306-313; dequantize_row_q4_K / q5_K / q6_K).  Quants per weight, scales per sub-block."""
    b = blocks.reshape(-1, refs.BLOCK[t][1]).astype(np.int64)
    nb = b.shape[0]
    f16 = lambda lo: (b[:, lo] | (b[:, lo + 1] << 8)).astype(np.uint16)
    q = np.zeros((nb, 256), np.int64)
    if t in (Q4_K, Q5_K):
        s = b[:, 4:16]
        sc = np.concatenate([s[:, 0:4] & 63, (s[:, 8:12] & 15) | ((s[:, 0:4] >> 6) << 4)], 1)
        mn = np.concatenate([s[:, 4:8] & 63, (s[:, 8:12] >> 4) | ((s[:, 4:8] >> 6) << 4)], 1)
        qs, qh = (b[:, 16:144], None) if t == Q4_K else (b[:, 48:176], b[:, 16:48])
        for j in range(4):
            q[:, 64 * j:64 * j + 32] = qs[:, 32 * j:32 * j + 32] & 15
            q[:, 64 * j + 32:64 * j + 64] = qs[:, 32 * j:32 * j + 32] >> 4
            if qh is not None:
                q[:, 64 * j:64 * j + 32] += ((qh >> (2 * j)) & 1) << 4
                q[:, 64 * j + 32:64 * j + 64] += ((qh >> (2 * j + 1)) & 1) << 4
        return sc, mn, q, f16(0), f16(2)
    ql, qh = b[:, 0:128], b[:, 128:192]
    for n in range(2):
        for j in range(4):
            lo = ql[:, 64 * n + 32 * (j & 1):64 * n + 32 * (j & 1) + 32] >> (4 * (j >> 1))
            q[:, 128 * n + 32 * j:128 * n + 32 * j + 32] = (lo & 15) | (((qh[:, 32 * n:32 * n + 32] >> (2 * j)) & 3) << 4)
    return blocks.reshape(nb, -1)[:, 192:208].view(np.int8).astype(np.int64), None, q, f16(208), None


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
@pytest.mark.parametrize("k,m", [(512, 48), (11008, 37)])
def test_edge_blocks_cover_every_scale_min_and_quant_edge(t, k, m):
    """refs.edge_blocks reaches what random_blocks (scales 32..63, mins = scales) and the reference-quantized pool (scales 26..63)
    do not: checked on the bytes, decoded as the reference decodes them, at the sizes the mat-mul tests draw."""
    w = refs.edge_blocks(t, k, m, seed=k + t)
    sc, mn, q, d, dmin = _decode_k_blocks(t, w)
    deq = np.zeros(w.size // refs.BLOCK[t][1] * 256, np.float32)
    getattr(refs.oracle(), "orc_dequantize_row_" + refs.TYPE_NAME[t])(ptr(w), ptr(deq), deq.size)
    assert np.isfinite(deq).all()
    nsub = sc.shape[1]
    scale_of = np.repeat(sc, 256 // nsub, axis=1)
    f = lambda h: h.view(np.float16).astype(np.float32)[:, None]
    if t == Q6_K:
        assert sorted(set(sc.ravel())) == list(range(-128, 128))
        want = f(d) * scale_of * (q - 32)
    else:
        assert sorted(set(sc.ravel())) == list(range(64)) and sorted(set(mn.ravel())) == list(range(64))
        assert (sc == mn).mean() < 0.05, "mins must be drawn independently of the scales"
        want = f(d) * scale_of * q - f(dmin) * np.repeat(mn, 32, axis=1)
    assert np.allclose(deq.reshape(want.shape), want, rtol=1e-6, atol=0), "decoder and the reference's dequantizer disagree"
    edges = {Q4_K: (0, 15), Q5_K: (0, 31, 15, 16), Q6_K: (0, 63, 15, 48)}[t]
    per_sub = q.reshape(q.shape[0], nsub, -1)
    for c in edges:   # whole sub-blocks of q = c: all bits clear, all set, only the low 4 or only the high bits set
        assert (per_sub == c).all(axis=2).any(), c
    for h in (d,) if dmin is None else (d, dmin):
        assert not ((h & 0x7c00) == 0x7c00).any(), "no inf or NaN"
        assert (h >> 15).any() and not (h >> 15).all(), "both signs"
        assert (((h & 0x7c00) == 0) & ((h & 0x3ff) != 0)).any(), "subnormal f16 values"


class TestAgainstCompiledReference:
    """Against what the compiled reference returned for the same inputs (tests/golden/reference_runs.npz)."""

    def test_quantizers_bit_exact(self):
        gold = refs.golden_runs()
        rng = np.random.default_rng(7)
        for trial in range(60):
            x = (rng.standard_normal(2048) * rng.choice([1e-3, 1, 50])).astype(np.float32)
            if trial % 7 == 0:
                x[256:512] = 0
            assert refs.digest(_oracle_quant(Q8_K, x)) == str(gold["act_quant_q8_K"][trial]), trial
            assert refs.digest(_oracle_quant(Q8_0, x)) == str(gold["act_quant_q8_0"][trial]), trial

    @pytest.mark.parametrize("t,at", TYPES)
    def test_vec_dot(self, t, at):
        o = refs.oracle()
        k = 4096
        wq = refs.reference_quantized_blocks(t, k, 16, seed=t).reshape(16, -1)
        act = _oracle_quant(at, np.random.default_rng(t).standard_normal(k).astype(np.float32))   # pinned by the test above
        fn = getattr(o, f"orc_vec_dot_{refs.TYPE_NAME[t]}_{'q8_K' if at == Q8_K else 'q8_0'}")
        want = refs.golden_runs()[f"vec_dot_{t}"]
        for i in range(16):
            b = np.float32(fn(k, ptr(wq[i]), ptr(act)))
            assert want[i].view(np.uint32) == b.view(np.uint32)

    def test_random_block_generator_is_valid_for_the_reference(self):
        """synth.random_blocks must produce blocks the reference dequantizes to finite, sensibly scaled weights (the oracle's
        dequantizers give the reference's bits: test_vec_dot_and_dequant_match_golden)."""
        from ctransformers_b200 import synth
        o = refs.oracle()
        for t in (Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K):
            blocks = np.ascontiguousarray(synth.random_blocks(t, 1024, 8, 0.02, np.random.default_rng(t)))
            out = np.zeros(8 * 1024, np.float32)
            getattr(o, "orc_dequantize_row_" + refs.TYPE_NAME[t])(ptr(blocks), ptr(out), out.size)
            assert refs.digest(out) == str(refs.golden_runs()[f"random_blocks_{t}_dequant"]), t
            assert np.isfinite(out).all()
            assert 0.01 < out.std() < 0.04, (t, out.std())
            assert abs(out.mean()) < 0.004


# ---- the whole-model restatement (oracle/llama_oracle.c) is pinned by the logits the reference produced
import modelcases  # noqa: E402


@pytest.mark.parametrize("name", list(modelcases.CASES))
def test_full_eval_matches_reference_golden(name, tmp_path_factory):
    gold = np.load(GOLD / f"model_{name}.npz")
    path, ctx = modelcases.build(name, tmp_path_factory.mktemp("orc"))
    m = refs.OracleModel(path, ctx)
    logits = m.eval(gold["prompt"].tolist()).copy()
    # bit-exact: the oracle reproduces the reference's fp32 accumulation order and FMA placement
    assert np.array_equal(logits.view(np.uint32), gold["first_logits"].view(np.uint32)), np.abs(logits - gold["first_logits"]).max()
    assert np.array_equal(m.embd.view(np.uint32), gold["first_embd"].view(np.uint32))
    toks = []
    for want in gold["tokens"][:6]:
        t = int(np.argmax(m.logits))
        toks.append(t)
        m.eval([t])
    assert toks == gold["tokens"][:6].tolist()


@pytest.mark.parametrize("key", list(modelcases.LONG_RUNS))
def test_long_context_runs_match_reference(key, tmp_path_factory):
    """The long-context runs of tests/test_long_context_gpu.py (contexts up to 8192, prompts up to 2280 tokens, chunks of 3 to
    512): the oracle's logits and hidden state after the prompt, greedy tokens and last logits are the reference's bits, so the
    GPU tests' comparisons with the oracle rest on the reference."""
    name, ctx, n_prompt, bs, n_new = modelcases.LONG_RUNS[key]
    path, _ = modelcases.build(name, tmp_path_factory.mktemp("orc_long"))
    first_logits, first_embd, toks, last_logits, _ = modelcases.oracle_greedy(refs.OracleModel(path, ctx), modelcases.seeded_prompt(name, n_prompt),
                                                                              n_new, bs)
    gold = refs.golden_runs()
    assert toks == gold[f"long_{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert refs.digest(v) == str(gold[f"long_{key}_{k}"]), k


@pytest.mark.parametrize("key", list(modelcases.REALQ_PREFILL))
def test_realq_prefill_runs_match_reference(key, tmp_path_factory):
    """The reference-quantized Q5_K_M runs of tests/test_model_gpu.py: the oracle gives the reference's bits, so the GPU test's
    comparison with the oracle rests on the reference."""
    arch, ftype = modelcases.REALQ_PREFILL[key]
    path = modelcases.build_realq(tmp_path_factory.mktemp("orc_realq"), arch, ftype)
    run = modelcases.oracle_greedy(refs.OracleModel(path, modelcases.REALQ_PREFILL_CTX), modelcases.realq_prompt(arch), modelcases.REALQ_PREFILL_NEW, 512)
    first_logits, first_embd, toks, last_logits, _ = run
    gold = refs.golden_runs()
    assert toks == gold[f"prefill_{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert refs.digest(v) == str(gold[f"prefill_{key}_{k}"]), k


@pytest.mark.parametrize("name", ["llama_tiny_q4km", "falcon_tiny_q5km"])
def test_full_eval_matches_live_reference_for_any_chunking(name, tmp_path_factory):
    """70-token prompt (so the V·P f16 dot uses both its SIMD part and its scalar tail), three chunkings, then 3 decode steps,
    against the reference's logits for the same run (tests/golden/reference_runs.npz)."""
    path, ctx = modelcases.build(name, tmp_path_factory.mktemp("orc_live"))
    ids = modelcases.long_prompt(name, bos=False)
    gold = refs.golden_runs()
    for bs in (8, 64, 33):
        m = refs.OracleModel(path, ctx)
        m.eval(ids, batch_size=bs)
        for step in range(3):
            assert refs.digest(m.logits) == str(gold[f"chunked_{name}_bs{bs}_logits"][step]), (bs, step)
            m.eval([int(np.argmax(m.logits))])
