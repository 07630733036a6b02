"""Q4_1 / Q5_1 weights and their Q8_1 activation, without a GPU: the plain-C restatement (oracle/q41_q51_oracle.c) against the
reference's known-answer vectors (golden/kat_q8_1.npz) and, where oracle/_ref is built, against the reference live; the forms the
restatement rejected against the same vectors; and the whole-model oracle against the reference's runs of the model cases."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import q41_q51_refs as Q
import refs

KAT = Q.GOLD / "kat_q8_1.npz"
SOURCES = ("refq", "pool", "edge")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("k", [32, 1024, 4544])
def test_quantize_row_q8_1_matches_reference_kat(k):
    g = np.load(KAT)
    for x, want in zip(g[f"x_{k}"], g[f"q81_{k}"]):
        assert np.array_equal(Q.quantize_q8_1(x), want)


def test_planted_rows_hold_what_they_claim():
    """All-zero blocks, the largest |x| first / in the middle / last, and products x*id exactly on a .5."""
    for x in Q.planted_rows(1024, seed=1):
        blk = x.reshape(-1, 32)
        amax = np.abs(blk).max(axis=1)
        assert (amax == 0).any()
        for at in (0, 13, 31):
            assert (np.argmax(np.abs(blk), axis=1) == at).any()
        nz = amax > 0
        prod = blk[nz] * (np.float32(127) / amax[nz])[:, None]
        assert (np.abs(prod - np.trunc(prod)) == 0.5).any()


@pytest.mark.parametrize("t", [Q.Q4_1, Q.Q5_1], ids=["q4_1", "q5_1"])
@pytest.mark.parametrize("src", SOURCES)
def test_vec_dot_and_dequantize_match_reference_kat(t, src):
    g = np.load(KAT)
    w, k = g[f"w_{src}_{t}"], g["dot_x"].shape[1]
    for a, x in enumerate(g["dot_x"]):
        act = Q.quantize_q8_1(x)
        got = np.array([Q.vec_dot(t, k, w[i], act) for i in range(len(w))], np.float32)
        assert np.array_equal(bits(got), bits(g[f"dot_{src}_{t}"][a]))
    deq = np.stack([Q.dequantize(t, w[i], k) for i in range(len(w))])
    assert np.array_equal(bits(deq), bits(g[f"deq_{src}_{t}"]))


def test_edge_blocks_reach_the_edges():
    for t in (Q.Q4_1, Q.Q5_1):
        b = Q.edge_blocks(t, 1024, 8, seed=t).reshape(-1, refs.BLOCK[t][1])
        d, m = b[:, 0:2].copy().view(np.float16)[:, 0], b[:, 2:4].copy().view(np.float16)[:, 0]
        for v in (d, m):
            assert (v > 0).any() and (v < 0).any() and (v == 0).any()
            assert ((np.abs(v) > 0) & (np.abs(v) < np.float16(6.1e-5))).any()      # fp16 subnormals
        q0 = 4 if t == Q.Q4_1 else 8
        assert (b[:, q0:] == 0).all(axis=1).any() and (b[:, q0:] == 0xFF).all(axis=1).any()
        if t == Q.Q5_1:
            qh = set(b[:, 4:8].copy().view("<u4")[:, 0].tolist())
            assert {0, 0xFFFFFFFF, 0x55555555, 0xAAAAAAAA, 0x0000FFFF, 0xFFFF0000} <= qh and len(qh) > 8


def test_rejected_forms_give_other_bits():
    """The vectors pin the reference's choices: an unfused summs chain, d_y rounded through fp16, or roundf instead of
    round-half-even each change some result."""
    g = np.load(KAT)
    for variant in (Q.DY_FP16, Q.ROUNDF):
        with refs.variant("orc_q1_set_variant", variant):
            assert any(not np.array_equal(Q.quantize_q8_1(x), want) for x, want in zip(g["x_1024"], g["q81_1024"])), variant
    for t in (Q.Q4_1, Q.Q5_1):
        w, k = g[f"w_refq_{t}"], 1024
        differ = 0
        for a, x in enumerate(g["dot_x"]):
            act = Q.quantize_q8_1(x)
            with refs.variant("orc_q1_set_variant", Q.SUMMS_UNFUSED):
                got = np.array([Q.vec_dot(t, k, w[i], act) for i in range(len(w))], np.float32)
            differ += int((bits(got) != bits(g[f"dot_refq_{t}"][a])).sum())
        assert differ > 0, t


def test_dequantize_forms_cannot_differ():
    """x*d + m fused or not: q*d (q in 0..31, d any finite fp16) is exact in fp32, so both forms round once and agree.  Checked
    for every finite fp16 d and every q, and the restatement's two forms agree on the known-answer blocks."""
    d = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)
    d = d[np.isfinite(d)].astype(np.float64)
    for q in range(32):
        p = q * d
        assert np.array_equal(p.astype(np.float32).astype(np.float64), p)
    g = np.load(KAT)
    for t in (Q.Q4_1, Q.Q5_1):
        for src in SOURCES:
            w = g[f"w_{src}_{t}"]
            for i in range(len(w)):
                with refs.variant("orc_q1_set_variant", Q.DEQ_UNFUSED):
                    unfused = Q.dequantize(t, w[i], 1024)
                assert np.array_equal(bits(unfused), bits(Q.dequantize(t, w[i], 1024)))


@pytest.mark.skipif(not refs.have_ref(), reason="oracle/_ref (the compiled reference) is not built here")
def test_against_live_reference():
    """Fresh seeded rows and blocks through the compiled reference: Q8_1 bytes, dots and dequantized rows, bit for bit."""
    rng = np.random.default_rng(77)
    for x in Q.planted_rows(2048, seed=77):
        assert np.array_equal(Q.quantize_q8_1(x), refs.ref_quantize_act(Q.Q8_1, x))
    for t in (Q.Q4_1, Q.Q5_1):
        for w in (Q.edge_blocks(t, 2048, 4, seed=5), Q.reference_quantized_blocks(t, 2048, 4, seed=6), Q.random_blocks(t, 2048, 4, seed=7)):
            w = w.reshape(4, -1)
            x = (rng.standard_normal(2048) * 3).astype(np.float32)
            act = refs.ref_quantize_act(Q.Q8_1, x)
            for i in range(4):
                assert np.float32(Q.vec_dot(t, 2048, w[i], act)) == np.float32(refs.ref_vec_dot(t, 2048, w[i], act))
            deq = np.zeros(4 * 2048, np.float32)
            refs.ref_traits(t)["to_float"](refs.ptr(np.ascontiguousarray(w)), refs.ptr(deq), deq.size)
            assert np.array_equal(bits(deq), bits(np.concatenate([Q.dequantize(t, w[i], 2048) for i in range(4)])))


def test_mul_mat_routes_other_types_to_the_original_oracle():
    """orc_mul_mat, which also takes Q4_1 / Q5_1, gives the reference's known answers for every other type (golden/kat_quant.npz:
    the reference's quantized weights dotted with its quantization of x)."""
    kat = np.load(refs.GOLD / "kat_quant.npz")
    for t in (refs.Q4_0, refs.Q5_0, refs.Q8_0, refs.Q4_K, refs.Q5_K, refs.Q6_K):
        w = kat[f"wq_{t}"]
        assert np.array_equal(bits(Q.mul_mat(t, w, kat["x_1024"], 1024, len(w))), bits(kat[f"dot_{t}"])), t


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("q41_q51_models")


def same_as_reference(key, run):
    gold = Q.golden_runs()
    first_logits, first_embd, toks, last_logits, _ = run
    assert toks == gold[f"{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert np.isfinite(v).all() and refs.digest(v) == str(gold[f"{key}_{k}"]), f"{k}: not the reference's bits"


@pytest.mark.parametrize("bs", Q.BATCH_SIZES)
@pytest.mark.parametrize("name", list(Q.model_cases()))
def test_whole_model_oracle_matches_reference(name, bs, model_dir):
    path, ctx = Q.build_model(name, model_dir)
    same_as_reference(f"{name}_bs{bs}", modelcases.oracle_greedy(refs.OracleModel(path, ctx), Q.prompt_for(name), Q.N_NEW, bs))


@pytest.mark.skipif(not refs.have_ref(), reason="oracle/_ref (the compiled reference) is not built here")
@pytest.mark.parametrize("name", ["llama_tiny_q4_1", "falcon_narrow_mixed"])
def test_whole_model_against_live_reference(name, model_dir):
    from ctransformers_b200 import AutoModelForCausalLM
    path, ctx = Q.build_model(name, model_dir)
    for bs in Q.BATCH_SIZES:
        llm = AutoModelForCausalLM.from_pretrained(str(path), lib=str(refs.REF_SO), context_length=ctx, threads=4)
        same_as_reference(f"{name}_bs{bs}", modelcases.run_greedy(llm, Q.prompt_for(name), Q.N_NEW, batch_size=bs))


def test_model_cases_have_the_promised_types(model_dir):
    """Which matrices each case holds in which type: the mixes the GPU tests rely on."""
    from ctransformers_b200 import synth
    want = {
        "llama_tiny_q4_1": {"attn_q": Q.Q4_1, "ffn_down": Q.Q4_1, "output": synth.Q6_K, "token_embd": Q.Q4_1},
        "falcon_narrow_q5_1": {"attn_qkv": Q.Q5_1, "ffn_down": Q.Q5_1, "output": synth.Q8_0, "token_embd": Q.Q5_1},
        "falcon_narrow_mixed": {"attn_qkv": Q.Q5_1, "ffn_up": Q.Q5_1, "ffn_down": synth.Q5_K, "output": synth.Q8_0},
        "llama_qkv_mixed": {"attn_q": Q.Q5_1, "attn_k": synth.Q4_0, "attn_v": Q.Q5_1},
    }
    for name, kinds in want.items():
        tensors = refs.read_gguf(Q.build_model(name, model_dir)[0])[1]
        for kind, t in kinds.items():
            names = [n for n in tensors if n.split(".")[-2] == kind]
            assert names and all(tensors[n][0] == t for n in names), (name, kind)
