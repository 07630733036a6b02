"""Shared definitions of the small synthetic models the end-to-end tests (and the golden generator) use."""
from pathlib import Path

import numpy as np

from ctransformers_b200 import synth

CASES = {
    # name: (arch, shape, ftype, ctx)
    "llama_tiny_q4km": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=3, n_ctx_train=256), "Q4_K_M", 96),
    "llama_gqa_q5km": ("llama", synth.LlamaShape(n_vocab=2048, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2816, n_layer=2, n_ctx_train=256), "Q5_K_M", 96),
    "llama_tiny_q4_0": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256), "Q4_0", 64),
    "llama_tiny_q8_0": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=2, n_head_kv=2, n_ff=512, n_layer=2, n_ctx_train=256), "Q8_0", 64),
    "falcon_tiny_q5km": ("falcon", synth.FalconShape(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=1, n_ff=2048, n_layer=2, n_ctx_train=256), "Q5_K_M", 96),
    # wide enough that every mat-vec launch has many row tiles per CTA and QKV mixes Q4_K with Q6_K (layer 0 "use_more_bits")
    "llama_wide_q4km": ("llama", synth.LlamaShape(n_vocab=1536, n_embd=2048, n_head=16, n_head_kv=16, n_ff=5632, n_layer=2, n_ctx_train=256), "Q4_K_M", 96),
    "llama_tiny_q5_0": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256), "Q5_0", 64),
    "falcon_tiny_q4_0": ("falcon", synth.FalconShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=1, n_ff=1024, n_layer=2, n_ctx_train=256), "Q4_0", 64),
}
PROMPT_LEN = 37   # with 24 new tokens the context reaches 61: the f16 dot of V·P then uses its SIMD lanes AND its scalar tail
N_NEW = 24


def build(name, directory, quantizer=None):
    arch, shape, ftype, ctx = CASES[name]
    path = Path(directory) / f"{name}.gguf"
    if not path.exists():
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=11, quantizer=quantizer)
    return path, ctx


def prompt_for(name):
    arch, shape, _, _ = CASES[name]
    rng = np.random.default_rng(5)
    lo = 259 if arch == "llama" else 0
    ids = rng.integers(lo, shape.n_vocab, PROMPT_LEN).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def long_prompt(name, bos=True):
    """70 tokens: three batched prefill launches (32 + 32 + 6), and a V·P f16 dot that uses both its SIMD part and its tail."""
    arch, shape, _, _ = CASES[name]
    ids = np.random.default_rng(9).integers(259 if arch == "llama" else 0, shape.n_vocab, 70).tolist()
    if bos and arch == "llama":
        ids[0] = 1
    return ids


def seeded_prompt(name, n, seed=17):
    """n seeded token ids for a model case (BOS first on llama): the prompts of the long-context runs."""
    arch, shape, _, _ = CASES[name]
    ids = np.random.default_rng(seed).integers(259 if arch == "llama" else 0, shape.n_vocab, n).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


# Long-context runs: key -> (model case, context_length, prompt tokens, batch_size, greedy steps).  What the engine does at each
# length (tests/test_long_context_gpu.py asserts it through ctb_llm_paths):
#   c2304_p1100  batched prefill (35 launches), then ring decode at T 1101..1124 (nchv 5, cv 3); with CTB_NO_PREFILL=1 the ring
#                step runs at every T from 1, through every cv step up to T = 1025
#   c2304_p2280  the context fills exactly: the last step attends over 2304 positions (V items fill the ring slot, cv 2)
#   c3072        the V items of 12 chunks do not fit the ring: attention reads K / V from global memory (attn_body in the step)
#   c1152_bs3    chunks of 3 tokens: every token's n_total is its chunk's end, past the token for the first two of each chunk
#   c4096        the batched kernel's attention scratch does not fit shared memory: no batched prefill
#   c8192        the attention scratch leaves room for one ring slot per consumer warp (10 slots)
LONG_RUNS = {
    "llama_tiny_q4km_c2304_p1100": ("llama_tiny_q4km", 2304, 1100, 512, 24),
    "falcon_tiny_q5km_c2304_p1100": ("falcon_tiny_q5km", 2304, 1100, 512, 24),
    "llama_gqa_q5km_c2304_p520": ("llama_gqa_q5km", 2304, 520, 512, 8),
    "llama_tiny_q4km_c2304_p2280": ("llama_tiny_q4km", 2304, 2280, 512, 24),
    "llama_tiny_q4km_c3072_p600": ("llama_tiny_q4km", 3072, 600, 512, 8),
    "llama_tiny_q4km_c1152_p1100_bs3": ("llama_tiny_q4km", 1152, 1100, 3, 4),
    "falcon_tiny_q5km_c4096_p300": ("falcon_tiny_q5km", 4096, 300, 64, 8),
    "llama_tiny_q4km_c8192_p300": ("llama_tiny_q4km", 8192, 300, 64, 8),
    "llama_tiny_q4km_c1024_p600": ("llama_tiny_q4km", 1024, 600, 512, 8),
}


def oracle_greedy(model, prompt, n_new, batch_size):
    """run_greedy's results from an oracle model (refs.OracleModel): greedy = the first largest logit."""
    model.eval(prompt, batch_size=batch_size)
    first_logits, first_embd = model.logits.copy(), model.embd.copy()
    toks = []
    for _ in range(n_new):
        toks.append(int(np.argmax(model.logits)))
        model.eval([toks[-1]])
    return first_logits, first_embd, toks, model.logits.copy(), None


REALQ_PROMPT = [1] + np.random.default_rng(0).integers(259, 1024, 30).tolist()


def build_realq(directory, arch="llama", ftype="Q4_K_M"):
    """A model whose weights are blocks of the reference's quantizer (refs.reference_quantized_blocks): Q4_K_M Llama by default."""
    import refs
    path = Path(directory) / ("realq.gguf" if (arch, ftype) == ("llama", "Q4_K_M") else f"realq_{arch}_{ftype.lower()}.gguf")
    if not path.exists():
        if arch == "llama":
            shape = synth.LlamaShape(n_vocab=1024, n_embd=512, n_head=4, n_head_kv=4, n_ff=1536, n_layer=2, n_ctx_train=128)
        else:
            shape = synth.FalconShape(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=1, n_ff=2048, n_layer=2, n_ctx_train=128)
        (synth.write_llama if arch == "llama" else synth.write_falcon)(
            path, shape, ftype, seed=3, sigma=0.05,
            quantizer=lambda t, w: refs.reference_quantized_blocks(t, w.shape[1], w.shape[0], seed=w.shape[0] * 7 + t))
    return path


# Reference-quantized Q5_K_M models through batched prefill: key -> (arch, ftype).  Their Q5_K blocks have mins that differ from
# their scales, which no random-block model has.  A 70-token prompt at batch_size 512: launches of 32 + 32 + 6 tokens.
REALQ_PREFILL = {"realq_llama_q5km": ("llama", "Q5_K_M"), "realq_falcon_q5km": ("falcon", "Q5_K_M")}
REALQ_PREFILL_CTX, REALQ_PREFILL_NEW = 96, 6


def realq_prompt(arch):
    ids = np.random.default_rng(9).integers(259 if arch == "llama" else 0, 1024, 70).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def run_greedy(llm, prompt, n_new, batch_size=8):
    """prompt eval (chunked like the reference default) then n_new greedy steps; returns logits after the prompt,
    embeddings after the prompt, the greedy tokens and the logits after the last step."""
    llm.eval(prompt, batch_size=batch_size)
    first_logits = np.array(llm.logits, dtype=np.float32)
    first_embd = np.array(llm.embeddings, dtype=np.float32)
    toks, gaps = [], []
    for _ in range(n_new):
        lg = np.array(llm.logits, dtype=np.float32)
        top2 = np.sort(lg)[-2:]
        gaps.append(float(top2[1] - top2[0]))
        t = llm.sample(top_k=1, repetition_penalty=1.0, seed=0)
        toks.append(int(t))
        llm.eval([t])
    return first_logits, first_embd, toks, np.array(llm.logits, dtype=np.float32), gaps


# Models whose token_embd (F32) holds rows that break the kernels' order of the first layer's norm sums (refs.norm_order_rows):
# model case -> norm mode.  Q4_K_M Llama: step kernel and batched prefill; Q4_0 Llama: k_matvec; Q5_K_M Falcon: LayerNorm, with
# rows that break Σx and rows that break Σ(x - mean)² alone.  The prompt is one 40-token chunk, which the batched prefill runs as
# a full 32-token launch and a short 8-token one, with planted tokens in both; then every planted token is a decode step of its
# own, then greedy steps.
NORM_ORDER_MODELS = {"llama_tiny_q4km": 1, "llama_tiny_q4_0": 1, "falcon_tiny_q5km": 2}
NORM_ORDER_PLANTED = list(range(300, 308))
NORM_ORDER_AT = [3, 17, 30, 33, 36, 39]   # prompt positions of planted tokens: 3 in the full launch, 3 in the short one
NORM_ORDER_PROMPT, NORM_ORDER_GREEDY = 40, 4


def build_norm_order(name, directory):
    import refs
    arch, shape, ftype, ctx = CASES[name]
    path = Path(directory) / f"{name}_norm_order.gguf"
    if not path.exists():
        rows, _, _ = refs.norm_order_rows(NORM_ORDER_MODELS[name], shape.n_embd, seed=shape.n_embd)
        rows = np.resize(rows, (len(NORM_ORDER_PLANTED), shape.n_embd))
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=11,
                                                                      token_rows=dict(zip(NORM_ORDER_PLANTED, rows)))
    return path, ctx


def norm_order_prompt(name):
    ids = seeded_prompt(name, NORM_ORDER_PROMPT, seed=23)
    for i, p in enumerate(NORM_ORDER_AT):
        ids[p] = NORM_ORDER_PLANTED[i % len(NORM_ORDER_PLANTED)]
    return ids


def norm_order_run(eval_fn, state_fn, pick_fn, name):
    """The prompt in one chunk, every planted token as a decode step, then greedy steps.  eval_fn(tokens, batch_size), state_fn()
    -> (logits, embeddings), pick_fn() -> greedy token.  Returns ([(logits, embeddings) after the prompt and after every step],
    greedy tokens)."""
    eval_fn(norm_order_prompt(name), 512)
    states = [state_fn()]
    for t in NORM_ORDER_PLANTED:
        eval_fn([t], 512)
        states.append(state_fn())
    toks = []
    for _ in range(NORM_ORDER_GREEDY):
        toks.append(int(pick_fn()))
        eval_fn([toks[-1]], 512)
        states.append(state_fn())
    return states, toks


def norm_order_llm_run(llm, name):
    return norm_order_run(lambda t, bs: llm.eval(t, batch_size=bs),
                          lambda: (np.array(llm.logits, np.float32), np.array(llm.embeddings, np.float32)),
                          lambda: llm.sample(top_k=1, repetition_penalty=1.0, seed=0), name)


def norm_order_oracle_run(model, name):
    return norm_order_run(lambda t, bs: model.eval(t, batch_size=bs), lambda: (model.logits.copy(), model.embd.copy()),
                          lambda: int(np.argmax(model.logits)), name)
