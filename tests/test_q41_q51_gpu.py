"""Q4_1 / Q5_1 on the GPU (k_matvec with a Q8_1 activation, Q4_1 / Q5_1 embedding rows), bit-exact with the oracle
(oracle/q41_q51_oracle.c) at op level, at Falcon-7B's real projection shapes among others, and with the reference's runs of the
model cases through the public Python API."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import q41_q51_refs as Q
import refs
from refs import ptr

pytestmark = pytest.mark.gpu
TYPES = pytest.mark.parametrize("t", [Q.Q4_1, Q.Q5_1], ids=["q4_1", "q5_1"])


def same(got, want, what=""):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ (max |d| {np.abs(got - want).max():.3e})"


def weights(src, t, k, m, seed):
    return {"random": Q.random_blocks, "refq": Q.reference_quantized_blocks, "edge": Q.edge_blocks}[src](t, k, m, seed)


@pytest.mark.parametrize("k", [32, 4096, 4544, 18176])
def test_quantize_row_q8_1(lib, k):
    for x in Q.planted_rows(k, seed=k):
        got = np.zeros(refs.row_bytes(Q.Q8_1, k), np.uint8)
        assert lib.ctb_quantize_row_q8_1(ptr(x), ptr(got), k) == 0
        assert np.array_equal(got, Q.quantize_q8_1(x))


@TYPES
@pytest.mark.parametrize("src", ["random", "refq", "edge"])
@pytest.mark.parametrize("K,M,N", [(32, 1, 1), (256, 3, 2), (4096, 64, 2), (11008, 33, 1),
                                   (4544, 4672, 1), (4544, 4544, 1), (4544, 18176, 1), (18176, 4544, 1)])   # last four: Falcon-7B qkv, wo, up, down
def test_mul_mat(lib, t, src, K, M, N):
    w = weights(src, t, K, M, seed=K + M + t)
    rng = np.random.default_rng(K * 3 + M)
    x = (rng.standard_normal(K * N) * rng.choice([0.01, 1.0, 30.0])).astype(np.float32)
    if K >= 64:
        x[32:64] = 0                                   # an all-zero Q8_1 block: d = s = 0
    got = np.zeros(M * N, np.float32)
    assert lib.ctb_mul_mat(t, ptr(w), ptr(x), ptr(got), K, M, N) == 0
    same(got, Q.mul_mat(t, w, x, K, M, N), f"type {t} {src} K {K} M {M}")


@TYPES
def test_ffn_gate(lib, t):
    K, M = 4544, 1536
    w1, w3 = Q.edge_blocks(t, K, M, seed=1), Q.reference_quantized_blocks(t, K, M, seed=2)
    x = np.random.default_rng(3).standard_normal(K).astype(np.float32)
    got = np.zeros(M, np.float32)
    assert lib.ctb_ffn_gate(t, ptr(w1), ptr(w3), ptr(x), ptr(got), K, M) == 0
    g, u = Q.mul_mat(t, w1, x, K, M), Q.mul_mat(t, w3, x, K, M)
    refs.oracle().orc_silu(ptr(g), ptr(g), M)
    same(got, g * u, f"type {t}")


@TYPES
@pytest.mark.parametrize("src", ["random", "refq", "edge"])
def test_get_row(lib, t, src):
    K, rows = 4544, 12
    table = weights(src, t, K, rows, seed=9 + t)
    rb = refs.row_bytes(t, K)
    for r in (0, 5, rows - 1):
        got = np.zeros(K, np.float32)
        assert lib.ctb_get_row(t, ptr(table), K, rows, r, ptr(got)) == 0
        same(got, Q.dequantize(t, table[r * rb:(r + 1) * rb], K), f"type {t} row {r}")


@TYPES
def test_prefill_mul_mat_refuses(lib, t):
    K, M = 256, 16
    w = Q.random_blocks(t, K, M, seed=1)
    x = np.zeros(K * 2, np.float32)
    out = np.zeros(M * 2, np.float32)
    types, rows, epi = (C.c_int * 1)(t), (C.c_int * 1)(M), (C.c_int * 1)(0)
    wp = (C.c_void_p * 1)(w.ctypes.data)
    rc = lib.ctb_prefill_mul_mat(1, types, wp, rows, K, 2, ptr(x), None, 0, None, None, 1e-5, epi, None, None, ptr(out), 64, 64, None)
    assert rc != 0


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("q41_q51_gpu_models")


PATH_FIELDS = ("fused", "ring_attn", "slots", "prefill_ok", "prefill_launches", "single_steps")


@pytest.mark.parametrize("bs", Q.BATCH_SIZES)
@pytest.mark.parametrize("name", list(Q.model_cases()))
def test_whole_model_against_reference(name, bs, model_dir):
    """Logits and embeddings after the prompt, 24 greedy tokens and the last logits: the reference's bits.  No batched prefill
    runs (it takes K-quant weights only): every prompt token goes through the single-token path."""
    from ctransformers_b200 import AutoModelForCausalLM
    path, ctx = Q.build_model(name, model_dir)
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    first_logits, first_embd, toks, last_logits, _ = modelcases.run_greedy(llm, Q.prompt_for(name), Q.N_NEW, batch_size=bs)
    gold, key = Q.golden_runs(), f"{name}_bs{bs}"
    assert toks == gold[f"{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert np.isfinite(v).all() and refs.digest(v) == str(gold[f"{key}_{k}"]), f"{k}: not the reference's bits"
    out = (C.c_int * len(PATH_FIELDS))()
    assert llm.ctb_llm_paths(out, len(PATH_FIELDS)) == len(PATH_FIELDS)
    paths = dict(zip(PATH_FIELDS, out))
    assert paths["prefill_ok"] == 0 and paths["prefill_launches"] == 0, paths


@pytest.mark.parametrize("name", ["llama_tiny_q4_1", "falcon_narrow_mixed", "llama_qkv_mixed"])
def test_whole_model_against_oracle(name, model_dir):
    """The same runs against the whole-model oracle, value by value (a failure shows where, not only that)."""
    from ctransformers_b200 import AutoModelForCausalLM
    path, ctx = Q.build_model(name, model_dir)
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    run = modelcases.run_greedy(llm, Q.prompt_for(name), 8, batch_size=8)
    want = modelcases.oracle_greedy(refs.OracleModel(path, ctx), Q.prompt_for(name), 8, 8)
    for i, what in ((0, "logits after the prompt"), (1, "embeddings after the prompt"), (3, "last logits")):
        same(run[i], want[i], what)
    assert run[2] == want[2]
