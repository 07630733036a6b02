"""Model cases whose attention heads are neither 64 nor 128 wide (test infrastructure, never the product).

Each case is a synthetic GGUF written from a seed; tests/golden/make_golden_head_dims.py runs it through the unmodified
reference and stores what it computed in golden/head_dims_runs.npz.  The oracle's whole-model attention can take a K·q tail
the reference does not use: refs.variant("orc_hd_set_variant", TAIL_FP32 or TAIL_IN_LANES).
"""
from pathlib import Path

import numpy as np

from refs import GOLD

N_NEW = 8
TAIL_FP32, TAIL_IN_LANES = 1, 2   # orc_hd_set_variant: the K·q tail summed in fp32, or folded into the SIMD lanes


def model_cases():
    """name -> (arch, shape, ftype, ctx, prompt length, batch sizes)."""
    from ctransformers_b200 import synth
    L, F = synth.LlamaShape, synth.FalconShape
    return {
        # legacy types: k_matvec and k_attn; n_embd 800 is not a multiple of 256, so the head is Q8_0
        "llama_hd100_q4_0": ("llama", L(n_vocab=1024, n_embd=800, n_head=8, n_head_kv=8, n_ff=1024, n_layer=2, n_ctx_train=256), "Q4_0", 128, 70, (8, 64, 5)),
        "llama_hd100_gqa_q4_0": ("llama", L(n_vocab=1024, n_embd=800, n_head=8, n_head_kv=2, n_ff=1024, n_layer=2, n_ctx_train=256), "Q4_0", 128, 70, (8, 64, 5)),
        # K-quants: step kernel, ring attention, batched prefill
        "llama_hd80_q4km_gqa": ("llama", L(n_vocab=1024, n_embd=1280, n_head=16, n_head_kv=4, n_ff=1536, n_layer=2, n_ctx_train=256), "Q4_K_M", 128, 70, (8, 64, 5)),
        "llama_hd96_q5km": ("llama", L(n_vocab=1024, n_embd=768, n_head=8, n_head_kv=8, n_ff=1536, n_layer=2, n_ctx_train=256), "Q5_K_M", 128, 70, (8, 64, 5)),
        "falcon_hd96_q5km_mqa": ("falcon", F(n_vocab=1024, n_embd=768, n_head=8, n_head_kv=1, n_ff=3072, n_layer=2, n_ctx_train=256), "Q5_K_M", 128, 70, (8, 64, 5)),
        # a long prompt: decode reads 20 K items of up to 57 rows (160 bytes each) per task from the step kernel's ring
        "llama_hd80_long": ("llama", L(n_vocab=1024, n_embd=1280, n_head=16, n_head_kv=4, n_ff=1536, n_layer=2, n_ctx_train=4096), "Q4_K_M", 2304, 1100, (512,)),
    }


# The OpenLLaMA-3B-shaped file (synth.OPENLLAMA_3B, 26 layers, 32 heads of 100, K = 3200 / 8640) in Q4_0 with a Q8_0 head, as
# the reference's quantizer writes such models: a 32-token prompt at batch_size 8, then 8 greedy steps.  Kept apart from
# model_cases(): the CPU oracle would take too long on it.
BIG_CASES = {"openllama3b_q4_0": ("llama", None, "Q4_0", 128, 32, (8,))}


def all_cases():
    from ctransformers_b200 import synth
    cases = dict(model_cases())
    for name, (arch, _, ftype, ctx, n, bss) in BIG_CASES.items():
        cases[name] = (arch, synth.OPENLLAMA_3B, ftype, ctx, n, bss)
    return cases


def kquant(name):
    return all_cases()[name][2].endswith("_M")


def build_model(name, directory):
    from ctransformers_b200 import synth
    arch, shape, ftype, ctx = all_cases()[name][:4]
    path = Path(directory) / f"{name}.gguf"
    if not path.exists():
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=13)
    return path, ctx


def prompt_for(name):
    arch, shape, _, _, n = all_cases()[name][:5]
    ids = np.random.default_rng(6).integers(259 if arch == "llama" else 0, shape.n_vocab, n).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def golden_runs():
    """What the reference computed on the model cases (golden/head_dims_runs.npz)."""
    return np.load(GOLD / "head_dims_runs.npz")
