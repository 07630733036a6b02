"""Attention heads that are neither 64 nor 128 wide (even sizes from 32 to 256), bit-exact with the reference: every attention
path at op level, RoPE, and whole models through the public API against the reference's runs (golden/head_dims_runs.npz)."""
import ctypes as C
import functools

import numpy as np
import pytest

import head_dims_refs as H
import modelcases
import refs
from refs import ptr

pytestmark = pytest.mark.gpu

ATTN_PATHS = {0: "k_attn", 1: "step_ring", 2: "step_global", 3: "prefill"}
# (n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, rope mode, hard), as test_ops_gpu.ATTN_CASES.  T crosses the K-item
# boundaries of each head size's ring geometry: ST_SLOT / (2 * k_stride(hd)) rows per item = 144 (hd 32), 57 (80), 48 (96),
# 44 (100), 41 (112), 18 (256).
ATTN_CASES = {
    "hd32-mha-T144-146": (8, 8, 32, 600, 143, 3, False, 0, 0, False),
    "hd32-mqa-neox-batch32": (8, 1, 32, 777, 500, 32, True, 0, 2, False),
    "hd80-gqa-T57-59": (16, 4, 80, 1100, 56, 3, False, 0, 0, False),
    "hd80-gqa-neox-T1000": (16, 4, 80, 2304, 998, 3, True, 0, 2, False),
    "hd80-ntotal-tail": (4, 4, 80, 1000, 39, 1, False, 20, 0, False),
    "hd96-mha-T48-50": (8, 8, 96, 513, 47, 3, False, 0, 0, False),
    "hd96-mqa-neox-batch32": (8, 1, 96, 999, 300, 32, True, 0, 2, False),
    "hd100-mha-T44-46": (8, 8, 100, 601, 43, 3, False, 0, 0, False),
    "hd100-gqa-T88-89": (8, 2, 100, 2304, 87, 2, False, 0, 0, False),
    "hd100-mqa-neox-straddle256": (8, 1, 100, 1025, 254, 5, True, 0, 2, False),
    "hd100-ntotal-chunk": (8, 8, 100, 2304, 700, 5, True, 57, 0, False),
    "hd100-full-ctx": (4, 4, 100, 2304, 2300, 4, False, 0, 0, False),
    "hd112-gqa-T41-43": (8, 2, 112, 3001, 40, 3, False, 0, 2, False),
    "hd112-mha-T1537": (4, 4, 112, 2000, 1536, 1, False, 0, 0, False),
    "hd256-gqa-T18-20": (4, 2, 256, 700, 17, 3, False, 0, 0, False),
    "hd256-mqa-neox-T513": (4, 1, 256, 2304, 512, 2, True, 0, 2, False),
    "hard-hd100": (8, 2, 100, 1500, 1200, 3, True, 0, 0, True),
    "hard-hd80": (8, 1, 80, 600, 300, 5, True, 0, 2, True),
    "hard-hd256": (4, 1, 256, 600, 100, 2, True, 0, 0, True),
}


def same_bits(got, want, what=""):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ (max |d| {np.abs(got - want).max():.3e})"


def _attn_inputs(n_head, n_kv, hd, n_ctx, pos0, n_tok, chunk, extra, mode, hard):
    rng = np.random.default_rng(n_head * 7919 + hd * 31 + n_ctx + pos0 * 3 + n_tok)
    q = rng.standard_normal((n_tok, n_head * hd)).astype(np.float32) * (40.0 if hard else 1.0)
    k = (rng.standard_normal((n_tok, n_kv * hd)) * 0.7).astype(np.float32)
    v = rng.standard_normal((n_tok, n_kv * hd)).astype(np.float32)
    kc = (rng.standard_normal((n_ctx, n_kv * hd)) * 0.7).astype(np.float16).view(np.uint16)
    vc = rng.standard_normal((n_kv * hd, n_ctx)).astype(np.float16).view(np.uint16)
    if hard:   # a whole channel group of V, the channels of a short last group and a few more are zero
        zero = list(range(32)) + [40, 77 % hd, hd - 1, hd - 3]
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
    """Output, K cache and V cache identical to the reference's attention block.  A path refuses a shape only by the library's
    own rule: the ring past 2304 positions (st_attn_ring_ok), the batched kernel at n_ctx >= 4096 or past 32 tokens."""
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
    same_bits(out, want, "output")
    assert np.array_equal(kc, want_kc), f"K cache: {int((kc != want_kc).sum())} entries differ"
    assert np.array_equal(vc, want_vc), f"V cache: {int((vc != want_vc).sum())} entries differ"


@pytest.mark.parametrize("hd", [264, 30, 99, 0])
def test_attention_path_refuses_other_head_sizes(lib, hd):
    n_head, n_kv, n_ctx, n_tok = 2, 2, 64, 1
    q = np.zeros((n_tok, n_head * max(hd, 1)), np.float32)
    k = np.zeros((n_tok, n_kv * max(hd, 1)), np.float32)
    kc = np.zeros((n_ctx, n_kv * max(hd, 1)), np.uint16)
    vc = np.zeros((n_kv * max(hd, 1), n_ctx), np.uint16)
    out = np.zeros_like(q)
    nt = np.array([1], np.int32)
    for path in ATTN_PATHS:
        assert lib.ctb_attention_path(path, ptr(q), ptr(k), ptr(k), ptr(kc), ptr(vc), ptr(out), n_head, n_kv, hd, n_ctx, 0, n_tok, ptr(nt), 0,
                                      10000.0, 0.1) == -1


@pytest.mark.parametrize("hd", [32, 80, 96, 100, 112, 256])
@pytest.mark.parametrize("mode", [0, 2])
def test_rope_bit_exact(lib, mode, hd):
    o = refs.oracle()
    rng = np.random.default_rng(hd * 3 + mode)
    for pos in (0, 1, 37, 511):
        x = rng.standard_normal((8, hd)).astype(np.float32)
        want, got = x.copy(), x.copy()
        o.orc_rope(ptr(want), 8, hd, pos, mode, 10000.0, 1.0)
        assert lib.ctb_rope(ptr(got), 8, hd, pos, mode, 10000.0, 1.0) == 0
        same_bits(got, want, f"pos {pos}")


@pytest.mark.parametrize("n_head,n_kv,T,n_total", [(4, 4, 1, 1), (8, 2, 300, 300), (8, 1, 45, 64), (4, 4, 1027, 1027)])
def test_attention_hd100_bit_exact(lib, n_head, n_kv, T, n_total):
    hd = 100
    o = refs.oracle()
    rng = np.random.default_rng(T + n_kv)
    q = rng.standard_normal((n_head, hd)).astype(np.float32)
    kc = (rng.standard_normal((T, n_kv, hd)) * 0.7).astype(np.float16)
    vt = rng.standard_normal((n_kv * hd, T)).astype(np.float16)
    scale = np.float32(1.0 / np.sqrt(np.float32(hd)))
    got = np.zeros((n_head, hd), np.float32)
    assert lib.ctb_attention(ptr(q), ptr(kc), ptr(vt), ptr(got), n_head, n_kv, hd, T, n_total, float(scale)) == 0
    want = np.zeros((n_head, hd), np.float32)
    vpad = np.zeros((n_kv * hd, n_total), np.float16)
    vpad[:, :T] = vt
    for h in range(n_head):
        kvh = h // (n_head // n_kv)
        kslice = np.ascontiguousarray(kc[:, kvh, :])
        vslice = np.ascontiguousarray(vpad[kvh * hd:(kvh + 1) * hd])
        o.orc_attn_head_n(ptr(q[h]), ptr(kslice), hd, ptr(vslice), n_total, hd, T, n_total, float(scale), ptr(want[h]))
    same_bits(got, want)


# ------------------------------------------------------------------------------------------------------ whole models
@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("head_dims_gpu_models")


PATH_FIELDS = ("fused", "ring_attn", "slots", "prefill_ok", "prefill_launches", "single_steps")
# every model case, and the OpenLLaMA-3B-shaped Q4_0 file (32-token prompt at batch_size 8 + 8 greedy steps)
RUNS = [(name, bs) for name, case in H.all_cases().items() for bs in case[5]]


@pytest.mark.parametrize("env", ["default", "no-prefill-no-fuse"])
@pytest.mark.parametrize("name,bs", RUNS, ids=[f"{n}-bs{b}" for n, b in RUNS])
def test_whole_model_against_reference(name, bs, env, model_dir, monkeypatch):
    """Logits and embeddings after the prompt, 8 greedy tokens and the last logits: the reference's bits, through the paths the
    model's weight types select.  The K-quant models run again without batched prefill and without the fused step kernel."""
    if env != "default":
        if not H.kquant(name):
            pytest.skip("legacy-type models take neither the batched prefill nor the step kernel")
        monkeypatch.setenv("CTB_NO_PREFILL", "1")
        monkeypatch.setenv("CTB_STEP_FUSE", "0")
    from ctransformers_b200 import AutoModelForCausalLM
    path, ctx = H.build_model(name, model_dir)
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    first_logits, first_embd, toks, last_logits, _ = modelcases.run_greedy(llm, H.prompt_for(name), H.N_NEW, batch_size=bs)
    gold, key = H.golden_runs(), f"{name}_bs{bs}"
    assert toks == gold[f"{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert np.isfinite(v).all() and refs.digest(v) == str(gold[f"{key}_{k}"]), f"{k}: not the reference's bits"
    out = (C.c_int * len(PATH_FIELDS))()
    assert llm.ctb_llm_paths(out, len(PATH_FIELDS)) == len(PATH_FIELDS)
    paths = dict(zip(PATH_FIELDS, out))
    if not H.kquant(name):   # k_matvec + k_attn: no step kernel (so no ring attention), no batched prefill
        assert paths["fused"] == 0 and paths["ring_attn"] == 0, paths
        assert paths["prefill_ok"] == 0 and paths["prefill_launches"] == 0, paths
    elif env == "default":
        assert paths["fused"] == 1 and paths["ring_attn"] == 1 and paths["prefill_ok"] == 1, paths
        if bs >= 32:
            assert paths["prefill_launches"] > 0, paths
    else:
        assert paths["fused"] == 0 and paths["prefill_launches"] == 0, paths


def test_head_size_outside_the_set_is_refused(model_dir, capfd):
    """hd 264 (2 heads of an F16 model of width 528): create fails at load, with the message."""
    from ctransformers_b200 import synth
    from ctransformers_b200.lib import load_library
    path = model_dir / "llama_hd264_f16.gguf"
    synth.write_llama(path, synth.LlamaShape(n_vocab=400, n_embd=528, n_head=2, n_head_kv=2, n_ff=256, n_layer=1, n_ctx_train=64), "F16", seed=1)
    from ctransformers_b200.lib import ConfigStruct
    lib = load_library()
    assert not lib.ctransformers_llm_create(str(path).encode(), b"gguf", ConfigStruct(64, 0, True, False))
    assert "unsupported head size 264" in capfd.readouterr().err
