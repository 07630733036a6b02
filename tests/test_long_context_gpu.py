"""GPU parity tests, whole path, at long contexts: prompts of hundreds to thousands of tokens, where the engine switches
between its attention implementations (step-kernel ring, step kernel from global memory, batched prefill, k_attn) and its
shared-memory layouts.  Each run is compared with the whole-model oracle run the same way (full vectors, readable diffs) and
with the digests of what the reference computed for it (tests/golden/reference_runs.npz, keys long_<run>_*).  Every test
also asserts, through ctb_llm_paths, which implementations the run took: a change of a threshold or a switch that reroutes
a run fails here instead of quietly testing something else.

Bar: identical bits, as everywhere in this suite."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import refs

pytestmark = pytest.mark.gpu
PATH_FIELDS = ("fused", "ring_attn", "slots", "prefill_ok", "prefill_launches", "single_steps")


def same_bits(what, got, want):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} values differ from the oracle, max |diff| {np.abs(got - want).max():.3e}"


def paths(llm):
    out = (C.c_int * len(PATH_FIELDS))()
    assert llm.ctb_llm_paths(out, len(PATH_FIELDS)) == len(PATH_FIELDS)
    return dict(zip(PATH_FIELDS, out))


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("long_models")


_oracle_runs = {}


def oracle_run(key, model_dir):
    """The oracle's results for a LONG_RUNS entry, computed once per module (most of this file's time is this CPU work)."""
    if key not in _oracle_runs:
        name, ctx, n_prompt, bs, n_new = modelcases.LONG_RUNS[key]
        path, _ = modelcases.build(name, model_dir)
        _oracle_runs[key] = modelcases.oracle_greedy(refs.OracleModel(path, ctx), modelcases.seeded_prompt(name, n_prompt), n_new, bs)
    return _oracle_runs[key]


def load_run(key, model_dir):
    from ctransformers_b200 import AutoModelForCausalLM
    name, ctx, n_prompt, bs, n_new = modelcases.LONG_RUNS[key]
    path, _ = modelcases.build(name, model_dir)
    return AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx), modelcases.seeded_prompt(name, n_prompt), n_new, bs


def check(key, run, model_dir):
    first_logits, first_embd, toks, last_logits, _ = run
    o_first, o_embd, o_toks, o_last, _ = oracle_run(key, model_dir)
    same_bits("logits after the prompt", first_logits, o_first)
    same_bits("hidden state after the prompt", first_embd, o_embd)
    assert toks == o_toks, "greedy tokens"
    same_bits("logits after the last step", last_logits, o_last)
    gold = refs.golden_runs()
    assert toks == gold[f"long_{key}_tokens"].tolist()
    for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
        assert refs.digest(v) == str(gold[f"long_{key}_{k}"]), f"{k}: not the reference's bits"


# key, environment, what ctb_llm_paths must report after the run (prefill_launches: exact; single_steps: a lower bound)
MATRIX = {
    # 1100 tokens at batch_size 512 = chunks 512 + 512 + 76 = 16 + 16 + 3 batched launches; decode T 1101..1124 on the ring
    # (nchv 5, cv 3)
    "ring-decode-after-prefill": ("llama_tiny_q4km_c2304_p1100", {}, dict(fused=1, ring_attn=1, slots=20, prefill_ok=1, prefill_launches=35)),
    "falcon-ring-decode-after-prefill": ("falcon_tiny_q5km_c2304_p1100", {}, dict(fused=1, ring_attn=1, slots=20, prefill_ok=1, prefill_launches=35)),
    "gqa-hd128": ("llama_gqa_q5km_c2304_p520", {}, dict(fused=1, ring_attn=1, slots=20, prefill_ok=1, prefill_launches=17)),
    # every T from 1 to 1124 on the ring step: every cv transition up to T = 1025
    "ring-decode-every-T": ("llama_tiny_q4km_c2304_p1100", {"CTB_NO_PREFILL": "1"},
                            dict(fused=1, ring_attn=1, slots=20, prefill_ok=0, prefill_launches=0, single_steps=1100)),
    # 2280 + 24 positions: the context is full at the last step (V items fill the ring slot: nchv 9, cv 2)
    "context-full": ("llama_tiny_q4km_c2304_p2280", {}, dict(fused=1, ring_attn=1, slots=20, prefill_ok=1, prefill_launches=72)),
    # 12 V chunks do not fit the ring: the step kernel reads K / V from global memory; the batched prefill still fits
    "no-ring": ("llama_tiny_q4km_c3072_p600", {}, dict(fused=1, ring_attn=0, slots=20, prefill_ok=1, prefill_launches=19)),
    # chunks of 3 tokens: batch_eval hands the engine the whole prompt, so its consecutive positions still go through the
    # batched kernel (35 launches), each token with the n_total of its own 3-token chunk ...
    "prefill-chunks-of-3": ("llama_tiny_q4km_c1152_p1100_bs3", {}, dict(fused=1, ring_attn=1, slots=20, prefill_ok=1, prefill_launches=35)),
    # ... and without it, single-token steps with n_total > T
    "single-token-chunks-of-3": ("llama_tiny_q4km_c1152_p1100_bs3", {"CTB_NO_PREFILL": "1"},
                                 dict(fused=1, ring_attn=1, slots=20, prefill_ok=0, prefill_launches=0, single_steps=1100)),
    # the batched kernel's per-warp attention scratch does not fit shared memory: the prompt runs token by token
    "no-prefill-ctx4096": ("falcon_tiny_q5km_c4096_p300", {}, dict(fused=1, ring_attn=0, slots=20, prefill_ok=0, prefill_launches=0, single_steps=300)),
    # the attention scratch leaves room for one slot per consumer warp
    "step-ring-depth1": ("llama_tiny_q4km_c8192_p300", {}, dict(fused=1, ring_attn=0, slots=10, prefill_ok=0, prefill_launches=0, single_steps=300)),
    "ring-attn-depth1": ("llama_tiny_q4km_c1024_p600", {"CTB_ST_SLOTS": "10", "CTB_NO_PREFILL": "1"},
                         dict(fused=1, ring_attn=1, slots=10, prefill_ok=0, prefill_launches=0, single_steps=600)),
    # one kernel per op: the decode steps run k_attn
    "k_attn-decode": ("llama_tiny_q4km_c2304_p1100", {"CTB_STEP_FUSE": "0"}, dict(fused=0, ring_attn=0, slots=20, prefill_ok=1, prefill_launches=35)),
}


@pytest.mark.parametrize("row", list(MATRIX))
def test_long_context_against_oracle_and_reference(row, model_dir, monkeypatch):
    key, env, expect = MATRIX[row]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    llm, prompt, n_new, bs = load_run(key, model_dir)
    run = modelcases.run_greedy(llm, prompt, n_new, batch_size=bs)
    got = paths(llm)
    for k, v in expect.items():
        assert (got[k] >= v) if k == "single_steps" else (got[k] == v), f"{k}: {got}"
    check(key, run, model_dir)


def test_graph_decode_at_long_context(model_dir):
    """ctb_llm_decode_greedy (the CUDA-graph loop the benchmark times) after an 1100-token prompt: the oracle's tokens and, after
    24 steps, its logits."""
    key = "llama_tiny_q4km_c2304_p1100"
    llm, prompt, n_new, bs = load_run(key, model_dir)
    llm.eval(prompt, batch_size=bs)
    first = llm.sample(top_k=1, repetition_penalty=1.0)
    out = (C.c_int * n_new)()
    assert llm.ctb_llm_decode_greedy(first, len(prompt), n_new, out) > 0
    assert paths(llm)["ring_attn"] == 1
    _, _, o_toks, o_last, _ = oracle_run(key, model_dir)
    assert [first] + list(out[:n_new - 1]) == o_toks
    same_bits("logits after the last step", np.array(llm.logits, np.float32), o_last)
