"""Checkers for the Q3_K weight type (test infrastructure, never the product).

  * oracle helpers   the Q3_K dot, dequantizer and mat-mul of the one oracle library (refs.oracle())
  * block pools      ``reference_quantized_blocks`` (the reference quantizer's blocks, golden/q3k_blocks.npz) and ``edge_blocks``
  * model cases      synthetic GGUF files in the Q3_K presets; tests/golden/make_golden_q3k.py stores what the unmodified
                     reference computed on them in golden/q3k_runs.npz
"""
from pathlib import Path

import numpy as np

import refs
from refs import GOLD, Q3_K, ptr

SCALE_FOLD_IN_FLOAT = 1   # orc_q3k_set_variant: a fold order the reference does not use


def quantize_q8_k(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(refs.row_bytes(refs.Q8_K, x.size), np.uint8)
    refs.oracle().orc_quantize_row_q8_K(ptr(x), ptr(out), x.size)
    return out


def vec_dot(k, wrow, act):
    return float(refs.oracle().orc_vec_dot_q3_K_q8_K(k, ptr(np.ascontiguousarray(wrow)), ptr(np.ascontiguousarray(act))))


def dequantize(blocks, k):
    out = np.zeros(k, np.float32)
    refs.oracle().orc_dequantize_row_q3_K(ptr(np.ascontiguousarray(blocks)), ptr(out), k)
    return out


def mul_mat(t, w, x, K, M, N=1):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(M * N, np.float32)
    assert refs.oracle().orc_mul_mat(t, ptr(np.ascontiguousarray(w)), ptr(x), ptr(out), K, M, N) == 0
    return out


# -------------------------------------------------------------------------------------------------------- weight blocks
def reference_quantized_blocks(k, m, seed):
    """m rows of k Q3_K weights drawn from the blocks the reference's quantizer wrote (golden/q3k_blocks.npz)."""
    pool = np.load(GOLD / "q3k_blocks.npz")["blocks"]
    idx = np.random.default_rng(seed).integers(0, len(pool), m * (k // 256))
    return np.ascontiguousarray(pool[idx].reshape(-1))


F16_MAX, F16_MIN_SUB = 0x7BFF, 0x0001


def edge_blocks(k, m, seed):
    """m rows of k Q3_K weights at the edges of the format, cycling over the block index: random; all sixteen scales -32 (six-bit
    0); all +31 (63); hmask all 0 (every weight gets -4); hmask all 1; qs all 0; qs all 3; all three extremes at once (every
    v = (q - 4)(sc - 32) = 128).  d is an f16 edge value (refs._f16_edge: both signs, subnormals, zero) in most blocks, +-65504
    or the smallest subnormal in the rest."""
    rng = np.random.default_rng(seed)
    nb = m * (k // 256)
    out = rng.integers(0, 256, (nb, 110), dtype=np.uint8)
    kind = np.arange(nb) % 8
    out[kind == 1, 96:108] = 0x00
    out[kind == 2, 96:108] = 0xFF
    out[kind == 3, 0:32] = 0x00
    out[kind == 4, 0:32] = 0xFF
    out[kind == 5, 32:96] = 0x00
    out[kind == 6, 32:96] = 0xFF
    out[kind == 7, 0:108] = 0x00
    d = refs._f16_edge(rng, nb)
    pick = rng.integers(0, 6, nb)
    d[pick == 0] = F16_MAX
    d[pick == 1] = F16_MAX | 0x8000
    d[pick == 2] = F16_MIN_SUB | (rng.integers(0, 2, int((pick == 2).sum())).astype(np.uint16) << 15)
    out[:, 108:110] = d.view(np.uint8).reshape(nb, 2)
    return np.ascontiguousarray(out.reshape(-1))


def random_blocks(k, m, seed, sigma=0.02):
    from ctransformers_b200 import synth
    return np.ascontiguousarray(synth.random_blocks(Q3_K, k, m, sigma, np.random.default_rng(seed)))


def blocks(src, k, m, seed):
    return {"random": random_blocks, "refq": reference_quantized_blocks, "edge": edge_blocks}[src](k, m, seed)


# ------------------------------------------------------------------------------------------------------------ model cases
def model_cases():
    """name -> (arch, shape, ftype, ctx, prompt length, batch sizes, weights): weights "random" (synth.random_blocks) or
    "reference" (the Q3_K matrices from the reference quantizer's pool)."""
    from ctransformers_b200 import synth
    L, F = synth.LlamaShape, synth.FalconShape
    return {
        "llama_tiny_q3ks": ("llama", L(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256), "Q3_K_S", 128, 70,
                            (8, 64, 5), "random"),
        "llama_gqa_q3km": ("llama", L(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=2, n_ff=1024, n_layer=3, n_ctx_train=256), "Q3_K_M", 128, 70,
                           (8, 64, 5), "random"),
        "llama_q3kl": ("llama", L(n_vocab=1024, n_embd=512, n_head=4, n_head_kv=4, n_ff=1280, n_layer=2, n_ctx_train=256), "Q3_K_L", 128, 70,
                       (8, 64, 5), "random"),
        # 5 layers: ffn_down is Q5_K in layers 0-1, Q4_K where use_more_bits holds (2, 4) and Q3_K in layer 3; Q8_0 head
        "falcon_mqa_q3km": ("falcon", F(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=1, n_ff=2048, n_layer=5, n_ctx_train=256), "Q3_K_M", 128, 70,
                            (8, 64, 5), "random"),
        "llama_realq_q3ks": ("llama", L(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=8, n_ff=1024, n_layer=2, n_ctx_train=256), "Q3_K_S", 128, 70,
                             (8, 64, 5), "reference"),
        # heads of 80: the k_step<false, true> instantiation
        "llama_hd80_q3km": ("llama", L(n_vocab=1024, n_embd=1280, n_head=16, n_head_kv=4, n_ff=1536, n_layer=2, n_ctx_train=256), "Q3_K_M", 128, 70,
                            (8, 64, 5), "random"),
        # a long prompt: 1100 tokens at context 2304
        "llama_long_q3km": ("llama", L(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=2, n_ff=1024, n_layer=2, n_ctx_train=4096), "Q3_K_M", 2304, 1100,
                            (512,), "random"),
    }


# The 7B-shaped Q3_K_M file (synth.LLAMA2_7B, 3.3 GB): a 32-token prompt at batch_size 8, then 8 greedy steps.  Kept apart from
# model_cases(): the CPU oracle would take too long on it.
BIG_CASES = {"llama7b_q3km": ("llama", None, "Q3_K_M", 128, 32, (8,), "random")}
N_NEW = 8


def all_cases():
    from ctransformers_b200 import synth
    cases = dict(model_cases())
    for name, (arch, _, ftype, ctx, n, bss, w) in BIG_CASES.items():
        cases[name] = (arch, synth.LLAMA2_7B, ftype, ctx, n, bss, w)
    return cases


def build_model(name, directory):
    from ctransformers_b200 import synth
    arch, shape, ftype, ctx, _, _, weights = all_cases()[name]
    path = Path(directory) / f"{name}.gguf"
    if not path.exists():
        quantizer = None
        if weights == "reference":
            def quantizer(t, w):   # the Q3_K matrices from the pool; the others random
                if t != Q3_K:
                    return synth.random_blocks(t, w.shape[1], w.shape[0], 0.02, np.random.default_rng(w.shape[0] * 7 + t))
                return reference_quantized_blocks(w.shape[1], w.shape[0], seed=w.shape[0] * 7 + t)
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=17, quantizer=quantizer)
    return path, ctx


def prompt_for(name):
    arch, shape, _, _, n = all_cases()[name][:5]
    ids = np.random.default_rng(8).integers(259 if arch == "llama" else 0, shape.n_vocab, n).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def golden_runs():
    """What the reference computed on the model cases (golden/q3k_runs.npz)."""
    return np.load(GOLD / "q3k_runs.npz")
