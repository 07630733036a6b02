"""Q3_K on the GPU (the step kernel's block code, the batched prefill, embedding rows), bit-exact with the oracle
(oracle/q3k_oracle.c) at op level and with the reference's runs of the model cases through the public Python API."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import q3k_refs as Q
import refs
from refs import ptr

pytestmark = pytest.mark.gpu
SRCS = ["random", "refq", "edge"]


def same(got, want, what=""):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ (max |d| {np.abs(got - want).max():.3e})"


@pytest.mark.parametrize("src", SRCS)
@pytest.mark.parametrize("K,M,N", [(256, 1, 1), (256, 3, 2), (512, 17, 1), (1024, 16, 1), (1280, 33, 1), (2304, 40, 1), (4096, 64, 2),
                                   (11008, 45, 1), (4096, 22016, 1)])   # K = 1 .. 9 blocks: every chunk remainder of 5-block items
def test_mul_mat(lib, src, K, M, N):
    w = Q.blocks(src, K, M, seed=K + M)
    rng = np.random.default_rng(K * 3 + M)
    x = (rng.standard_normal(K * N) * rng.choice([0.01, 1.0, 30.0])).astype(np.float32)
    if K >= 512:
        x[256:512] = 0                                 # an all-zero Q8_K block
    got = np.zeros(M * N, np.float32)
    assert lib.ctb_mul_mat(Q.Q3_K, ptr(w), ptr(x), ptr(got), K, M, N) == 0
    same(got, Q.mul_mat(Q.Q3_K, w, x, K, M, N), f"{src} K {K} M {M}")


def test_mul_mat_fixtures(lib):
    """The stored reference dots: the Q8_K activations of the fixture rows are what the kernel's quantizer makes of dot_x."""
    kat = np.load(Q.GOLD / "q3k_kat.npz")
    K = kat["dot_x"].shape[1]
    for src in SRCS:
        w = np.ascontiguousarray(kat[f"w_{src}"])
        for j, x in enumerate(kat["dot_x"]):
            got = np.zeros(len(w), np.float32)
            assert lib.ctb_mul_mat(Q.Q3_K, ptr(w), ptr(np.ascontiguousarray(x)), ptr(got), K, len(w), 1) == 0
            same(got, kat[f"dot_{src}"][j], f"{src} row {j}")


def _prefill(lib, types, ws, rows, K, n_tok, x):
    nseg = len(types)
    out = np.zeros((n_tok, sum(rows)), np.float32)
    wp = (C.c_void_p * nseg)(*[w.ctypes.data for w in ws])
    rc = lib.ctb_prefill_mul_mat(nseg, (C.c_int * nseg)(*types), wp, (C.c_int * nseg)(*rows), K, n_tok, ptr(x), None, 0, None, None, 1e-5,
                                 (C.c_int * nseg)(*([0] * nseg)), None, None, ptr(out), 128, 64, None)
    assert rc == 0
    return out


@pytest.mark.parametrize("n_tok", [1, 5, 32])
@pytest.mark.parametrize("mix", ["q3k", "q3k_q4k_q6k"])
def test_prefill_mul_mat(lib, n_tok, mix):
    K = 2304
    types = [Q.Q3_K] if mix == "q3k" else [Q.Q3_K, refs.Q4_K, refs.Q6_K]
    rows = [70] if mix == "q3k" else [40, 33, 24]
    ws = []
    for s, (t, m) in enumerate(zip(types, rows)):
        if t == Q.Q3_K:
            ws.append(Q.blocks(("edge", "refq", "random")[n_tok % 3], K, m, seed=s + n_tok))
        else:
            ws.append(refs.edge_blocks(t, K, m, seed=s + n_tok))
    x = (np.random.default_rng(n_tok).standard_normal((n_tok, K)) * 2).astype(np.float32)
    got = _prefill(lib, types, ws, rows, K, n_tok, x)
    want = np.concatenate([Q.mul_mat(t, w, x, K, m, n_tok).reshape(n_tok, m) for t, w, m in zip(types, ws, rows)], axis=1)
    same(got, want, mix)


def test_ffn_gate(lib):
    K, M = 4096, 1100   # (edge blocks' d of 65504 would make the product inf or NaN, whose payload says nothing)
    w1, w3 = Q.random_blocks(K, M, seed=1), Q.reference_quantized_blocks(K, M, seed=2)
    x = np.random.default_rng(3).standard_normal(K).astype(np.float32)
    got = np.zeros(M, np.float32)
    assert lib.ctb_ffn_gate(Q.Q3_K, ptr(w1), ptr(w3), ptr(x), ptr(got), K, M) == 0
    g, u = Q.mul_mat(Q.Q3_K, w1, x, K, M), Q.mul_mat(Q.Q3_K, w3, x, K, M)
    refs.oracle().orc_silu(ptr(g), ptr(g), M)
    same(got, g * u)


@pytest.mark.parametrize("src", SRCS)
def test_get_row(lib, src):
    K, rows = 4096, 12
    table = Q.blocks(src, K, rows, seed=9)
    rb = refs.row_bytes(Q.Q3_K, K)
    for r in (0, 5, rows - 1):
        got = np.zeros(K, np.float32)
        assert lib.ctb_get_row(Q.Q3_K, ptr(table), K, rows, r, ptr(got)) == 0
        same(got, Q.dequantize(table[r * rb:(r + 1) * rb], K), f"row {r}")


def test_matvec_partition(lib):
    n_sm = 132
    first, meta = (C.c_int * (n_sm + 1))(), (C.c_int * 8)()
    assert lib.ctb_matvec_partition((C.c_int * 1)(Q.Q3_K), (C.c_int * 1)(22016), 1, 4096, n_sm, first, meta) == 0
    kb = (meta[7] >> 24) & 0xFF
    assert kb * 16 * 110 <= meta[1] and (meta[7] & 0xFFFFFF) == (4 | 3 << 8 | 2 << 16)
    assert first[0] == 0 and first[n_sm] == 22016 // 16 == meta[3]
    assert meta[6] >= -(-meta[3] // n_sm) * -(-16 // kb)
    assert lib.ctb_matvec_partition((C.c_int * 3)(Q.Q3_K, refs.Q4_K, refs.Q6_K), (C.c_int * 3)(4096, 1024, 1024), 3, 4096, n_sm, first, meta) == 0


# ------------------------------------------------------------------------------------------------------ whole models
@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("q3k_gpu_models")


PATH_FIELDS = ("fused", "ring_attn", "slots", "prefill_ok", "prefill_launches", "single_steps")
RUNS = [(name, bs) for name, case in Q.all_cases().items() for bs in case[5]]


@pytest.mark.parametrize("env", ["default", "no-prefill-no-fuse"])
@pytest.mark.parametrize("name,bs", RUNS, ids=[f"{n}-bs{b}" for n, b in RUNS])
def test_whole_model_against_reference(name, bs, env, model_dir, monkeypatch):
    """Logits and embeddings after the prompt, 8 greedy tokens and the last logits: the reference's bits, with batched prefill
    and the fused step kernel, and again without either."""
    if env != "default":
        if name in Q.BIG_CASES:
            pytest.skip("the 7B-shaped file runs once")
        monkeypatch.setenv("CTB_NO_PREFILL", "1")
        monkeypatch.setenv("CTB_STEP_FUSE", "0")
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
    if env == "default":
        assert paths["fused"] == 1 and paths["ring_attn"] == 1 and paths["prefill_ok"] == 1, paths
        if bs >= 32:
            assert paths["prefill_launches"] > 0, paths
        if Q.all_cases()[name][0] == "llama":
            assert llm.ctb_llm_launches_per_token() == 1
    else:
        assert paths["fused"] == 0 and paths["prefill_launches"] == 0, paths
    if name in Q.BIG_CASES:
        path.unlink()


@pytest.mark.parametrize("name", ["llama_gqa_q3km", "falcon_mqa_q3km"])
def test_whole_model_against_oracle(name, model_dir):
    """The same runs against the whole-model oracle, value by value (a failure shows where, not only that)."""
    from ctransformers_b200 import AutoModelForCausalLM
    path, ctx = Q.build_model(name, model_dir)
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    run = modelcases.run_greedy(llm, Q.prompt_for(name), 8, batch_size=64)
    want = modelcases.oracle_greedy(refs.OracleModel(path, ctx), Q.prompt_for(name), 8, 64)
    for i, what in ((0, "logits after the prompt"), (1, "embeddings after the prompt"), (3, "last logits")):
        same(run[i], want[i], what)
    assert run[2] == want[2]


def test_q2k_file_is_refused(model_dir, capfd):
    """A tensor in Q2_K (type 10): create fails at load, with the message."""
    from ctransformers_b200 import synth
    from ctransformers_b200.lib import ConfigStruct, load_library
    path = model_dir / "llama_q2k.gguf"
    synth.BLOCK.setdefault(10, (256, 84))
    try:
        synth.write_llama(path, synth.LlamaShape(n_vocab=400, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=1, n_ctx_train=64), "Q3_K_S",
                          seed=1, quantizer=lambda t, w: np.zeros(refs.row_bytes(t, w.shape[1]) * w.shape[0] if t != 10 else w.shape[0] * 84, np.uint8),
                          tensor_types={"ffn_up": 10})
    finally:
        synth.BLOCK.pop(10)
    lib = load_library()
    assert not lib.ctransformers_llm_create(str(path).encode(), b"gguf", ConfigStruct(64, 0, True, False))
    assert "quantization type 10 is not supported by the CUDA path" in capfd.readouterr().err
