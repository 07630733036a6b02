"""Q3_K on the CPU: the oracle's restatement (oracle/q3k_oracle.c) against what the unmodified reference computed
(golden/q3k_kat.npz, q3k_runs.npz), and a check that those stored results tell the reference's fp32 order from another."""
import numpy as np
import pytest

import modelcases
import q3k_refs as Q
import refs

SRCS = ["random", "refq", "edge"]


@pytest.fixture(scope="module")
def kat():
    return np.load(Q.GOLD / "q3k_kat.npz")


@pytest.mark.parametrize("src", SRCS)
def test_vec_dot_equals_reference(kat, src):
    w, acts, want = kat[f"w_{src}"], kat["dot_q8k"], kat[f"dot_{src}"]
    k = kat["dot_x"].shape[1]
    got = np.array([[Q.vec_dot(k, w[i], a) for i in range(len(w))] for a in acts], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{int((got != want).sum())} dots differ"


@pytest.mark.parametrize("src", SRCS)
def test_dequantize_equals_reference(kat, src):
    w, want = kat[f"w_{src}"], kat[f"deq_{src}"]
    got = np.stack([Q.dequantize(w[i], want.shape[1]) for i in range(len(w))])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_oracle_quantizes_activations_as_the_reference(kat):
    for x, want in zip(kat["dot_x"], kat["dot_q8k"]):
        assert np.array_equal(Q.quantize_q8_k(x), want)


def test_fixtures_tell_the_fold_order_apart(kat):
    """Each sub-block's scale times its integer sum taken in float and added to the lane (a fold the reference does not do)
    gives other bits on the stored dots: the fixtures can tell the orders apart."""
    k = kat["dot_x"].shape[1]
    differ = 0
    for src in SRCS:
        w, want = kat[f"w_{src}"], kat[f"dot_{src}"]
        with refs.variant("orc_q3k_set_variant", Q.SCALE_FOLD_IN_FLOAT):
            for j, a in enumerate(kat["dot_q8k"]):
                for i in range(len(w)):
                    differ += np.float32(Q.vec_dot(k, w[i], a)).view(np.uint32) != want[j, i].view(np.uint32)
    assert differ > 0


def test_edge_blocks_reach_the_extremes():
    w = Q.edge_blocks(2048, 4, seed=1).reshape(-1, 110)
    assert (w[:, 96:108] == 0).all(axis=1).any() and (w[:, 96:108] == 0xFF).all(axis=1).any()
    assert (w[:, 0:32] == 0).all(axis=1).any() and (w[:, 0:32] == 0xFF).all(axis=1).any()
    assert (w[:, 32:96] == 0).all(axis=1).any() and (w[:, 32:96] == 0xFF).all(axis=1).any()
    d = w[:, 108:110].copy().view(np.uint16).ravel()
    assert {0x7BFF, 0xFBFF} <= set(d.tolist()) and ((d & 0x7C00) == 0).any()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("q3k_models")


SMALL = [(name, bs) for name, case in Q.model_cases().items() if case[4] <= 70 for bs in case[5]]


@pytest.mark.parametrize("name,bs", SMALL, ids=[f"{n}-bs{b}" for n, b in SMALL])
def test_whole_model_oracle_equals_reference(name, bs, model_dir):
    """The whole-model oracle on the small cases gives the reference's stored digests at the same chunkings."""
    path, ctx = Q.build_model(name, model_dir)
    first_logits, first_embd, toks, last_logits, _ = modelcases.oracle_greedy(refs.OracleModel(path, ctx), Q.prompt_for(name), Q.N_NEW, bs)
    gold, key = Q.golden_runs(), f"{name}_bs{bs}"
    assert toks == gold[f"{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert refs.digest(v) == str(gold[f"{key}_{k}"]), k


def test_synth_q3k_presets_follow_the_reference_rules(model_dir):
    from ctransformers_b200 import synth
    L = synth.LlamaShape(n_vocab=400, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=8, n_ctx_train=64)
    F = synth.FalconShape(n_vocab=400, n_embd=256, n_head=4, n_head_kv=1, n_ff=512, n_layer=8, n_ctx_train=64)
    tt = lambda fn, sh, ft: getattr(synth, fn)(model_dir / "rules.gguf", sh, ft, seed=1)["tensor_types"]
    Q3, Q4, Q5, Q6, Q8 = synth.Q3_K, synth.Q4_K, synth.Q5_K, synth.Q6_K, synth.Q8_0
    s = tt("write_llama", L, "Q3_K_S")
    assert set(s.values()) == {Q3, Q6} and s["output.weight"] == Q6 and s["token_embd.weight"] == Q3
    m = tt("write_llama", L, "Q3_K_M")
    assert [m[f"blk.{i}.attn_v.weight"] for i in range(8)] == [Q5, Q5] + [Q4] * 6
    assert [m[f"blk.{i}.ffn_down.weight"] for i in range(8)] == [Q5, Q5] + [Q4] * 6
    assert m["blk.3.attn_output.weight"] == Q4 and m["blk.3.attn_q.weight"] == Q3 and m["blk.3.ffn_up.weight"] == Q3
    lg = tt("write_llama", L, "Q3_K_L")
    assert lg["blk.5.attn_v.weight"] == Q5 and lg["blk.5.ffn_down.weight"] == Q5 and lg["blk.5.attn_output.weight"] == Q5
    fm = tt("write_falcon", F, "Q3_K_M")
    more = [synth.use_more_bits(i, 8) for i in range(8)]
    assert [fm[f"blk.{i}.ffn_down.weight"] for i in range(8)] == [Q5, Q5] + [Q4 if more[i] else Q3 for i in range(2, 8)]
    assert fm["blk.4.attn_qkv.weight"] == Q4 and fm["blk.4.attn_output.weight"] == Q3 and fm["output.weight"] == Q8
    fl = tt("write_falcon", F, "Q3_K_L")
    assert fl["blk.4.ffn_down.weight"] == Q4 and fl["blk.4.attn_output.weight"] == Q4 and fl["blk.4.attn_qkv.weight"] == Q4
