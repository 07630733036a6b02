"""Checkers for the Q4_1 / Q5_1 weights and their Q8_1 activation (test infrastructure, never the product).

  * oracle helpers  the Q8_1 quantizer and the Q4_1 / Q5_1 dots, dequantizers and mat-mul of the one oracle library
                    (refs.oracle())
  * block pools     ``reference_quantized_blocks`` / ``edge_blocks`` for types 3 and 7, like refs.py's for the other types
"""
from pathlib import Path

import numpy as np

import refs
from refs import GOLD, Q4_1, Q5_1, Q8_1, ptr

# orc_q1_set_variant bits: the forms the reference does not use
SUMMS_UNFUSED, DEQ_UNFUSED, DY_FP16, ROUNDF = 1, 2, 4, 8


def quantize_q8_1(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(refs.row_bytes(Q8_1, x.size), np.uint8)
    refs.oracle().orc_quantize_row_q8_1(ptr(x), ptr(out), x.size)
    return out


def vec_dot(t, k, wrow, act):
    o = refs.oracle()
    return float((o.orc_vec_dot_q4_1_q8_1 if t == Q4_1 else o.orc_vec_dot_q5_1_q8_1)(k, ptr(np.ascontiguousarray(wrow)), ptr(act)))


def dequantize(t, blocks, k):
    blocks = np.ascontiguousarray(blocks)
    out = np.zeros(k, np.float32)
    o = refs.oracle()
    (o.orc_dequantize_row_q4_1 if t == Q4_1 else o.orc_dequantize_row_q5_1)(ptr(blocks), ptr(out), k)
    return out


def mul_mat(t, w, x, K, M, N=1):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(M * N, np.float32)
    assert refs.oracle().orc_mul_mat(t, ptr(np.ascontiguousarray(w)), ptr(x), ptr(out), K, M, N) == 0
    return out


# ------------------------------------------------------------------------------------------------------ activation rows
def planted_rows(k, seed):
    """Rows of k activations for the Q8_1 quantizer: seeded normals at several magnitudes, with all-zero blocks, blocks whose
    largest |x| sits at the first, a middle or the last element, and blocks where x*id lands exactly on a .5 (there
    round-half-even and roundf differ: x = (j + 0.5) * amax / 127 with amax a power of two, so x*id is exact)."""
    rng = np.random.default_rng(seed)
    rows = []
    for scale in (1e-3, 1.0, 40.0):
        x = (rng.standard_normal(k) * scale).astype(np.float32)
        nb = k // 32
        for b in range(nb):
            blk = x[32 * b:32 * b + 32]
            kind = b % 6
            if kind == 0:
                blk[:] = 0
            elif kind in (1, 2, 3):
                at = {1: 0, 2: 13, 3: 31}[kind]
                i = int(np.argmax(np.abs(blk)))
                blk[at], blk[i] = blk[i], blk[at]
                blk[at] = np.float32(np.abs(blk).max() * 1.5 * (1 if rng.integers(2) else -1))
            elif kind in (4, 5):
                amax = np.float32(2.0 ** int(rng.integers(-6, 6)))
                j = rng.integers(0, 126, 32)
                blk[:] = ((j + 0.5) * amax / 127.0).astype(np.float32) * rng.choice([-1, 1], 32).astype(np.float32)
                blk[int(rng.integers(0, 32))] = amax
        rows.append(x)
    return np.stack(rows)


# -------------------------------------------------------------------------------------------------------- weight blocks
def reference_quantized_blocks(t, k, m, seed):
    """m rows of k weights of type t, drawn from the blocks the reference's quantizer wrote (golden/q41_q51_blocks.npz)."""
    bs, sz = refs.BLOCK[t]
    pool = np.load(GOLD / "q41_q51_blocks.npz")[f"blocks_{t}"]
    idx = np.random.default_rng(seed).integers(0, len(pool), m * (k // bs))
    return np.ascontiguousarray(pool[idx].reshape(-1))


def edge_blocks(t, k, m, seed):
    """m rows of k weights of type t at the edges of the format: d and m of both signs, fp16 subnormals and zeros (m = 0 in
    about a tenth of the blocks), whole blocks of all-0 or all-15 nibbles, and for Q5_1 qh drawn from every pattern class
    (all clear, all set, alternating, random)."""
    rng = np.random.default_rng(seed)
    bs, sz = refs.BLOCK[t]
    nb = m * (k // bs)
    out = rng.integers(0, 256, (nb, sz), dtype=np.uint8)
    out[:, 0:2] = refs._f16_edge(rng, nb).view(np.uint8).reshape(nb, 2)
    out[:, 2:4] = refs._f16_edge(rng, nb).view(np.uint8).reshape(nb, 2)
    q0 = 4 if t == Q4_1 else 8
    kind = np.arange(nb) % 5
    out[kind == 1, q0:] = 0x00
    out[kind == 2, q0:] = 0xFF
    if t == Q5_1:
        pats = np.array([0x00000000, 0xFFFFFFFF, 0x55555555, 0xAAAAAAAA, 0x0000FFFF, 0xFFFF0000], np.uint32)
        sel = rng.integers(0, len(pats) + 2, nb)
        qh = np.where(sel < len(pats), pats[np.minimum(sel, len(pats) - 1)], rng.integers(0, 2 ** 32, nb, dtype=np.uint64).astype(np.uint32))
        out[:, 4:8] = qh.astype("<u4").view(np.uint8).reshape(nb, 4)
    return np.ascontiguousarray(out.reshape(-1))


def random_blocks(t, k, m, seed, sigma=0.02):
    from ctransformers_b200 import synth
    return np.ascontiguousarray(synth.random_blocks(t, k, m, sigma, np.random.default_rng(seed)))


# ------------------------------------------------------------------------------------------------------------ model cases
def _shapes():
    from ctransformers_b200 import synth
    llama = synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256)
    # Falcon-7B's proportions at test size: n_embd 320 = 5 x 64 (head_dim 64, MQA), n_ff 1280 = 5 x 256; no row length but
    # n_ff is a multiple of 256, as 4544 and 18176 are not / are
    falcon = synth.FalconShape(n_vocab=1024, n_embd=320, n_head=5, n_head_kv=1, n_ff=1280, n_layer=2, n_ctx_train=256)
    return llama, falcon


def model_cases():
    """name -> (arch, shape, ftype, tensor_types, ctx, weights): weights "random" (synth.random_blocks) or "reference" (blocks of
    the reference's quantizer, reference_quantized_blocks)."""
    from ctransformers_b200 import synth
    llama, falcon = _shapes()
    return {
        "llama_tiny_q4_1": ("llama", llama, "Q4_1", None, 64, "random"),            # Q4_1 body on k_matvec, Q6_K head on the step kernel
        "llama_tiny_q5_1": ("llama", llama, "Q5_1", None, 64, "random"),
        "falcon_narrow_q5_1": ("falcon", falcon, "Q5_1", None, 64, "random"),      # Q8_0 head, Q5_1 token_embd
        "falcon_narrow_mixed": ("falcon", falcon, "Q5_1", {"ffn_down": synth.Q5_K}, 64, "random"),   # step-kernel ffn_down
        "llama_realq_q5_1": ("llama", llama, "Q5_1", None, 64, "reference"),
        "llama_qkv_mixed": ("llama", llama, "Q5_1", {"attn_k": synth.Q4_0}, 64, "random"),          # QKV: a Q8_1 and a Q8_0 launch
    }


PROMPT_LEN, N_NEW = 37, 24
BATCH_SIZES = (8, 64, 5)


def build_model(name, directory):
    from ctransformers_b200 import synth
    arch, shape, ftype, types, ctx, weights = model_cases()[name]
    path = Path(directory) / f"{name}.gguf"
    if not path.exists():
        quantizer = None
        if weights == "reference":
            def quantizer(t, w):   # the Q5_1 matrices from the pool; the Q6_K head random (the K-quant pool's scales reach 2)
                if t not in (Q4_1, Q5_1):
                    return synth.random_blocks(t, w.shape[1], w.shape[0], 0.04, np.random.default_rng(w.shape[0] * 7 + t))
                return reference_quantized_blocks(t, w.shape[1], w.shape[0], seed=w.shape[0] * 7 + t)
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=11, quantizer=quantizer, tensor_types=types)
    return path, ctx


def prompt_for(name):
    arch, shape = model_cases()[name][:2]
    ids = np.random.default_rng(5).integers(259 if arch == "llama" else 0, shape.n_vocab, PROMPT_LEN).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def golden_runs():
    """What the reference computed on the model cases (golden/q41_q51_runs.npz, tests/golden/make_golden_q41_q51.py)."""
    return np.load(GOLD / "q41_q51_runs.npz")
