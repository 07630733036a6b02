"""Synthetic GGUF models (no network, no checkpoints): Llama- and Falcon-shaped files the reference loader accepts.

Two ways to fill a quantized tensor:
  * ``quantizer=None`` (default, fast): draw VALID random quant blocks directly — random nibbles / scales with
    fp16 super-scales chosen so the dequantized weights have a target standard deviation.  A 7B-shaped
    Q4_K_M file (3.8 GB) is produced in seconds.  Used by bench.py, smoke() and the large-shape tests.
  * ``quantizer=callable(ggml_type, f32_rows) -> bytes``: quantize real f32 weights with a caller-supplied
    quantizer (the tests pass the reference's own ggml_quantize_chunk from oracle/_ref).

Required keys / tensor names follow the reference loader (models/ggml/llama.cpp:1546-1642 hparams,
1648-1760 vocab incl. the mandatory <0xNN> byte tokens, 294-327 tensor names, 1878-2012 shapes).
The tensor-type mix of "Q4_K_M"/"Q5_K_M" follows the reference quantizer's rules (llama.cpp:4723-4725
use_more_bits, 4785-4829): output.weight and the more-bits attn_v / ffn_down in Q6_K, the rest Q4_K/Q5_K;
Falcon: output.weight Q8_0 (llama.cpp:4787-4789); "Q4_1"/"Q5_1": every matrix in the main type, output.weight Q6_K, or
Q8_0 where its rows are not whole 256-element blocks (llama.cpp:4785-4791); "Q3_K_S"/"Q3_K_M"/"Q3_K_L": Q3_K with the
per-tensor exceptions of llama.cpp:4793-4850 (_layer_types), token_embd in Q3_K.
"""
import struct
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, Optional

import numpy as np

F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q3_K, Q4_K, Q5_K, Q6_K = 0, 1, 2, 3, 6, 7, 8, 11, 12, 13, 14
BLOCK = {F32: (1, 4), F16: (1, 2), Q4_0: (32, 18), Q4_1: (32, 20), Q5_0: (32, 22), Q5_1: (32, 24), Q8_0: (32, 34), Q3_K: (256, 110),
         Q4_K: (256, 144), Q5_K: (256, 176), Q6_K: (256, 210)}

# gguf value types
_U32, _F32, _STR, _ARR, _I32 = 4, 6, 8, 9, 5


def tensor_nbytes(t, ne0, rows):
    be, bb = BLOCK[t]
    assert ne0 % be == 0, (t, ne0)
    return ne0 // be * bb * rows


# ------------------------------------------------------------------------------------------- writer
class GGUFWriter:
    """Minimal GGUF v2 writer (layout: models/ggml/ggml.c:19561-19800 reader)."""

    def __init__(self, path, alignment=32):
        self.path, self.align = Path(path), alignment
        self.kv, self.tensors = [], []

    @staticmethod
    def _s(s):
        b = s.encode() if isinstance(s, str) else bytes(s)
        return struct.pack("<Q", len(b)) + b

    def add_u32(self, k, v): self.kv.append(self._s(k) + struct.pack("<II", _U32, int(v)))
    def add_f32(self, k, v): self.kv.append(self._s(k) + struct.pack("<If", _F32, float(v)))
    def add_str(self, k, v): self.kv.append(self._s(k) + struct.pack("<I", _STR) + self._s(v))

    def add_arr_str(self, k, vals):
        self.kv.append(self._s(k) + struct.pack("<IIQ", _ARR, _STR, len(vals)) + b"".join(self._s(v) for v in vals))

    def add_arr_f32(self, k, vals):
        a = np.asarray(vals, dtype="<f4")
        self.kv.append(self._s(k) + struct.pack("<IIQ", _ARR, _F32, a.size) + a.tobytes())

    def add_arr_i32(self, k, vals):
        a = np.asarray(vals, dtype="<i4")
        self.kv.append(self._s(k) + struct.pack("<IIQ", _ARR, _I32, a.size) + a.tobytes())

    def add_tensor(self, name, ggml_type, shape, producer):
        """shape = (ne0, ne1) with ne0 contiguous; producer() -> bytes-like of exactly tensor_nbytes."""
        self.tensors.append((name, ggml_type, tuple(int(x) for x in shape), producer))

    def write(self):
        head = struct.pack("<IIQQ", 0x46554747, 2, len(self.tensors), len(self.kv)) + b"".join(self.kv)
        infos, off = [], 0
        for name, t, shape, _ in self.tensors:
            nb = tensor_nbytes(t, shape[0], int(np.prod(shape[1:])) if len(shape) > 1 else 1)
            infos.append(self._s(name) + struct.pack("<I", len(shape)) + b"".join(struct.pack("<Q", d) for d in shape) + struct.pack("<IQ", t, off))
            off += -(-nb // self.align) * self.align
        meta = head + b"".join(infos)
        pad = -len(meta) % self.align
        with open(self.path, "wb") as f:
            f.write(meta + b"\0" * pad)
            for name, t, shape, producer in self.tensors:
                nb = tensor_nbytes(t, shape[0], int(np.prod(shape[1:])) if len(shape) > 1 else 1)
                data = producer()
                data = memoryview(np.ascontiguousarray(data)).cast("B") if isinstance(data, np.ndarray) else memoryview(data)
                assert len(data) == nb, (name, len(data), nb)
                f.write(data)
                f.write(b"\0" * (-nb % self.align))
        return self.path


# ------------------------------------------------------------------------- random valid quant blocks
def _f16_bytes(vals):
    return np.asarray(vals, dtype=np.float16).view(np.uint8).reshape(len(vals), 2)


def random_blocks(t, ne0, rows, sigma, rng):
    """uint8 array of tensor_nbytes(t, ne0, rows) holding valid blocks whose dequantized weights have std ≈ sigma."""
    be, bb = BLOCK[t]
    n = ne0 // be * rows
    if t == F32:
        return (rng.standard_normal(n, dtype=np.float32) * sigma).view(np.uint8)
    if t == F16:
        return (rng.standard_normal(n, dtype=np.float32) * sigma).astype(np.float16).view(np.uint8)
    out = rng.integers(0, 256, size=(n, bb), dtype=np.uint8)   # quant payloads: any byte pattern is valid
    jitter = rng.uniform(0.7, 1.3, size=n)
    if t == Q4_0:      # w = d * (q - 8), q uniform 0..15 (std 4.61)
        out[:, 0:2] = _f16_bytes(sigma / 4.61 * jitter)
    elif t == Q5_0:    # w = d * (q - 16), q uniform 0..31 (std 9.23)
        out[:, 0:2] = _f16_bytes(sigma / 9.23 * jitter)
    elif t == Q8_0:    # w = d * q, q uniform int8 (std 73.9)
        out[:, 0:2] = _f16_bytes(sigma / 73.9 * jitter)
    elif t in (Q4_1, Q5_1):   # w = d * q + m, q uniform 0..15 (0..31); m = -c*d centres it; d (and so m) of either sign
        c, sq = (7.5, 4.61) if t == Q4_1 else (15.5, 9.23)
        d = sigma / sq * jitter * rng.choice([-1.0, 1.0], size=n)
        out[:, 0:2] = _f16_bytes(d)
        out[:, 2:4] = _f16_bytes(-c * d)
    elif t in (Q4_K, Q5_K):
        # w = d*sc*q - dmin*m.  Keep all 6-bit scales in [32,63] and m == sc, dmin = c*d with c = (qmax/2):
        # then w = d*sc*(q - c) is zero-mean with std ≈ d * 47.5 * std(q).
        c, sq = (7.5, 4.61) if t == Q4_K else (15.5, 9.23)
        d = sigma / (47.5 * sq) * jitter
        out[:, 0:2] = _f16_bytes(d)
        out[:, 2:4] = _f16_bytes(d * c)
        sc = rng.integers(32, 64, size=(n, 8), dtype=np.uint8)
        s = out[:, 4:16]
        s[:, 0:4] = (sc[:, 0:4] & 63) | ((sc[:, 4:8] >> 4) << 6)          # get_scale_min_k4 layout (k_quants.c:306-313)
        s[:, 4:8] = (sc[:, 0:4] & 63) | ((sc[:, 4:8] >> 4) << 6)          # mins identical to scales
        s[:, 8:12] = (sc[:, 4:8] & 0xF) | ((sc[:, 4:8] & 0xF) << 4)
    elif t == Q6_K:    # w = d * sc * (q - 32), q uniform 0..63 (std 18.5), sc int8
        sc = rng.integers(32, 128, size=(n, 16)).astype(np.int8)
        sc *= rng.choice(np.array([-1, 1], dtype=np.int8), size=(n, 16))
        out[:, 192:208] = sc.view(np.uint8)
        out[:, 208:210] = _f16_bytes(sigma / (18.5 * 85.0) * jitter)
    elif t == Q3_K:    # w = d * (sc - 32) * (q - 4), q uniform 0..7 (std 2.29); 6-bit scales in [0,8) u [56,64): |sc - 32| >= 24
        sc = rng.integers(0, 16, size=(n, 16), dtype=np.uint8)
        sc = np.where(sc < 8, sc, sc + 48).astype(np.uint8)
        s = out[:, 96:108]                                            # inverse of the unpacking in dequantize_row_q3_K (k_quants.c:593-598)
        s[:, 0:8] = (sc[:, 0:8] & 0xF) | ((sc[:, 8:16] & 0xF) << 4)
        s[:, 8:12] = (sc[:, 0:4] >> 4) | ((sc[:, 4:8] >> 4) << 2) | ((sc[:, 8:12] >> 4) << 4) | ((sc[:, 12:16] >> 4) << 6)
        out[:, 108:110] = _f16_bytes(sigma / (2.29 * 28.0) * jitter)
    else:
        raise ValueError(f"unsupported type {t}")
    return out.reshape(-1)


# ----------------------------------------------------------------------------------------- vocabulary
def make_spm_vocab(n_vocab):
    """<unk>,<s>,</s>, 256 byte tokens, then pieces: printable ASCII singles, '▁'-prefixed words, merges."""
    assert n_vocab >= 259 + 64
    toks, scores, types = ["<unk>", "<s>", "</s>"], [0.0, 0.0, 0.0], [2, 3, 3]
    for b in range(256):
        toks.append(f"<0x{b:02X}>"); scores.append(0.0); types.append(6)
    seen = set(toks)

    def add(piece, score):
        if piece not in seen and len(toks) < n_vocab:
            toks.append(piece); scores.append(float(score)); types.append(1); seen.add(piece)

    add("▁", -1.0)
    for ch in "etaoinshrdlucmfwypvbgkqjxzETAOINSHRDLUCMFWYPVBGKQJXZ0123456789.,!?'\"-:;()":
        add(ch, -5.0 - len(toks) * 1e-3)
    words = ["the", "of", "and", "to", "in", "is", "that", "it", "was", "for", "on", "are", "as", "with", "his", "they", "at", "be",
             "this", "from", "have", "or", "by", "one", "had", "not", "but", "what", "all", "were", "when", "we", "there", "can", "an",
             "your", "which", "their", "said", "if", "do", "will", "each", "about", "how", "up", "out", "them", "then", "she", "many",
             "some", "so", "these", "would", "other", "into", "has", "more", "her", "two", "like", "him", "see", "time", "could", "no",
             "make", "than", "first", "been", "its", "who", "now", "people", "my", "made", "over", "did", "down", "only", "way", "find",
             "use", "may", "water", "long", "little", "very", "after", "words", "called", "just", "where", "most", "know", "AI", "going"]
    for w in words:   # every prefix is a piece so the bigram merges can actually reach the word
        for k in range(2, len(w) + 1):
            add(w[:k], -3.0 - 0.01 * k)
        for k in range(1, len(w) + 1):
            add("▁" + w[:k], -2.0 - 0.01 * k)
    i = 0
    while len(toks) < n_vocab:
        add(f"▁tok{i}", -10.0 - i * 1e-4)
        i += 1
    return toks, scores, types


def make_bpe_vocab(n_vocab):
    """GPT-2 style vocabulary for Falcon GGUFs: the 256 raw single-byte strings (the reference BPE looks pieces up
    verbatim and dereferences a missing byte, llama.cpp:3316-3326, and it tokenizes "\\n" at load, llama.cpp:1748-1752),
    then merged pieces with their merge list, then fillers.  Tokens are returned as bytes."""
    toks = [bytes([b]) for b in range(256)]
    merges = []
    seen = set(toks)
    words = ["the", "of", "and", "to", "in", "is", "that", "it", "was", "for", "on", "are", "as", "with", "AI", "going", "be", "big",
             " the", " of", " and", " to", " in", " is", " that", " it", " was", " a", " be", " big", " going"]
    for w in words:
        wb = w.encode()
        for k in range(2, len(wb) + 1):
            piece = wb[:k]
            if piece not in seen:
                ga = lambda x: x.replace(b" ", "Ġ".encode())   # merges live in GPT-2's byte-level alphabet (llama.cpp:962-974)
                merges.append(ga(wb[:k - 1]) + b" " + ga(wb[k - 1:k]))
                toks.append(piece); seen.add(piece)
    i = 0
    while len(toks) < n_vocab:
        toks.append(f"<filler{i}>".encode()); i += 1
    toks = toks[:n_vocab]
    return toks, [0.0] * len(toks), [1] * len(toks), merges


# -------------------------------------------------------------------------------------------- models
def use_more_bits(i_layer, n_layer):
    return i_layer < n_layer // 8 or i_layer >= 7 * n_layer // 8 or (i_layer - n_layer // 8) % 3 == 2


@dataclass
class LlamaShape:
    n_vocab: int = 32000
    n_embd: int = 4096
    n_head: int = 32
    n_head_kv: int = 32
    n_ff: int = 11008
    n_layer: int = 32
    n_ctx_train: int = 4096
    rms_eps: float = 1e-5
    rope_base: float = 10000.0


LLAMA2_7B = LlamaShape()
LLAMA2_13B = LlamaShape(n_embd=5120, n_head=40, n_head_kv=40, n_ff=13824, n_layer=40)
# OpenLLaMA-3B and the models fine-tuned from it (the reference's MODEL_3B, 26 layers): heads of 100.  n_embd 3200 is not a
# multiple of 256, so the reference quantizer writes such files in the legacy types only.
OPENLLAMA_3B = LlamaShape(n_vocab=32000, n_embd=3200, n_head=32, n_head_kv=32, n_ff=8640, n_layer=26, n_ctx_train=2048)


@dataclass
class FalconShape:
    n_vocab: int = 65024
    n_embd: int = 4608      # Falcon-7B-shaped, K-quant clean (true 4544 is not a multiple of 256; SURVEY §8(d) note F1, option A)
    n_head: int = 72
    n_head_kv: int = 1
    n_ff: int = 18432
    n_layer: int = 32
    n_ctx_train: int = 2048
    eps: float = 1e-5


FALCON_7B_SHAPED = FalconShape()


def _type_plan(ftype):
    """(main type, more-bits type, output type, token_embd type) for a named ftype."""
    plan = {
        "Q4_K_M": (Q4_K, Q6_K, Q6_K, Q4_K), "Q5_K_M": (Q5_K, Q6_K, Q6_K, Q5_K), "Q4_0": (Q4_0, Q4_0, Q6_K, Q4_0), "Q5_0": (Q5_0, Q5_0, Q6_K, Q5_0),
        "Q4_1": (Q4_1, Q4_1, Q6_K, Q4_1), "Q5_1": (Q5_1, Q5_1, Q6_K, Q5_1),
        "Q8_0": (Q8_0, Q8_0, Q8_0, Q8_0), "Q6_K": (Q6_K, Q6_K, Q6_K, Q6_K), "Q4_K": (Q4_K, Q4_K, Q4_K, Q4_K),
        "Q5_K": (Q5_K, Q5_K, Q5_K, Q5_K), "F16": (F16, F16, F16, F16), "F32": (F32, F32, F32, F32),
        "Q3_K_S": (Q3_K, Q3_K, Q6_K, Q3_K), "Q3_K_M": (Q3_K, Q3_K, Q6_K, Q3_K), "Q3_K_L": (Q3_K, Q3_K, Q6_K, Q3_K),
    }
    return plan[ftype]


def _layer_types(ftype, falcon, il, n_layer):
    """{matrix kind: type} of layer il.  The Q3_K presets follow the reference quantizer's rules for QK_K = 256 and models
    other than 70B (llama.cpp:4793-4850); every other ftype puts attn_v / ffn_down in the more-bits type on use_more_bits layers."""
    main, more, _, _ = _type_plan(ftype)
    t = dict.fromkeys(("attn_q", "attn_k", "attn_v", "attn_output", "attn_qkv", "ffn_gate", "ffn_up", "ffn_down"), main)
    mb = use_more_bits(il, n_layer)
    if ftype == "Q3_K_M":
        t["attn_v"] = Q5_K if il < 2 else Q4_K
        t["ffn_down"] = Q5_K if il < 2 else (Q4_K if not falcon or mb else Q3_K)
        t["attn_output"] = Q3_K if falcon else Q4_K
        t["attn_qkv"] = Q4_K
    elif ftype == "Q3_K_L":
        t["attn_v"] = Q5_K
        t["ffn_down"] = Q4_K if falcon else Q5_K
        t["attn_output"] = Q4_K if falcon else Q5_K
        t["attn_qkv"] = Q4_K
    elif ftype != "Q3_K_S":
        t["attn_v"] = t["ffn_down"] = more if mb else main
    return t


def _weight_producer(t, ne0, rows, sigma, seed, quantizer: Optional[Callable]):
    def produce():
        rng = np.random.default_rng(seed)
        if quantizer is None or t in (F32, F16):
            return random_blocks(t, ne0, rows, sigma, rng)
        w = rng.standard_normal((rows, ne0), dtype=np.float32) * sigma
        return quantizer(t, w)
    return produce


def _f32_table(n_vocab, E, sigma, seed, token_rows):
    """token_embd as F32 rows: N(0, sigma²) values, with token_rows {token id: row [E]} in place of the drawn rows."""
    def produce():
        table = np.random.default_rng(seed).standard_normal((n_vocab, E), dtype=np.float32) * np.float32(sigma)
        for tok, row in token_rows.items():
            table[tok] = np.asarray(row, np.float32)
        return table
    return produce


def _output_type(out_t, n_embd):
    """The reference quantizer writes output.weight in Q8_0 where its rows are not whole K-quant blocks (llama.cpp:4785-4791)."""
    return Q8_0 if out_t in (Q3_K, Q4_K, Q5_K, Q6_K) and n_embd % 256 else out_t


def write_llama(path, shape: LlamaShape = LLAMA2_7B, ftype="Q4_K_M", seed=0, quantizer=None, sigma=0.02, emb_sigma=1.0, token_rows=None,
                tensor_types=None):
    """Llama-architecture GGUF.  Returns dict(path, weight_bytes_per_token, tensor_types).  token_rows {token id: row}: token_embd
    is written as F32 with these rows (the rest drawn), so a test can choose exactly what the first layer's norm sees.
    tensor_types {tensor kind, e.g. "attn_k": type}: that matrix of every layer in the given type instead of the ftype's."""
    _, _, out_t, emb_t = _type_plan(ftype)
    out_t = _output_type(out_t, shape.n_embd)
    tensor_types = tensor_types or {}
    w = GGUFWriter(path)
    a = "llama"
    w.add_str("general.architecture", a)
    w.add_str("general.name", f"synthetic-{a}-{ftype}")
    w.add_u32(f"{a}.context_length", shape.n_ctx_train)
    w.add_u32(f"{a}.embedding_length", shape.n_embd)
    w.add_u32(f"{a}.block_count", shape.n_layer)
    w.add_u32(f"{a}.feed_forward_length", shape.n_ff)
    w.add_u32(f"{a}.rope.dimension_count", shape.n_embd // shape.n_head)
    w.add_u32(f"{a}.attention.head_count", shape.n_head)
    w.add_u32(f"{a}.attention.head_count_kv", shape.n_head_kv)
    w.add_f32(f"{a}.attention.layer_norm_rms_epsilon", shape.rms_eps)
    if shape.rope_base != 10000.0:
        w.add_f32(f"{a}.rope.freq_base", shape.rope_base)
    toks, scores, types = make_spm_vocab(shape.n_vocab)
    w.add_str("tokenizer.ggml.model", "llama")
    w.add_arr_str("tokenizer.ggml.tokens", toks)
    w.add_arr_f32("tokenizer.ggml.scores", scores)
    w.add_arr_i32("tokenizer.ggml.token_type", types)
    w.add_u32("tokenizer.ggml.bos_token_id", 1)
    w.add_u32("tokenizer.ggml.eos_token_id", 2)
    w.add_u32("tokenizer.ggml.unknown_token_id", 0)

    E, FF, GQA = shape.n_embd, shape.n_ff, shape.n_embd // shape.n_head * shape.n_head_kv
    sid = [seed * 100003]
    per_token = [0]
    types_used = {}

    def mat(name, t, ne0, rows, sg, count=True):
        sid[0] += 1
        t = tensor_types.get(name.split(".")[-2], t)
        w.add_tensor(name, t, (ne0, rows), _weight_producer(t, ne0, rows, sg, sid[0], quantizer))
        types_used[name] = t
        if count:
            per_token[0] += tensor_nbytes(t, ne0, rows)

    def vec(name, n, base=1.0):
        sid[0] += 1
        s = sid[0]
        w.add_tensor(name, F32, (n,), lambda: (base + 0.1 * np.random.default_rng(s).standard_normal(n, dtype=np.float32)).astype(np.float32))

    if token_rows is None:
        mat("token_embd.weight", emb_t, E, shape.n_vocab, emb_sigma, count=False)
    else:
        sid[0] += 1
        w.add_tensor("token_embd.weight", F32, (E, shape.n_vocab), _f32_table(shape.n_vocab, E, emb_sigma, sid[0], token_rows))
        types_used["token_embd.weight"] = F32
    for il in range(shape.n_layer):
        b = f"blk.{il}."
        lt = _layer_types(ftype, False, il, shape.n_layer)
        vec(b + "attn_norm.weight", E)
        mat(b + "attn_q.weight", lt["attn_q"], E, E, sigma)
        mat(b + "attn_k.weight", lt["attn_k"], E, GQA, sigma)
        mat(b + "attn_v.weight", lt["attn_v"], E, GQA, sigma)
        mat(b + "attn_output.weight", lt["attn_output"], E, E, sigma)
        vec(b + "ffn_norm.weight", E)
        mat(b + "ffn_gate.weight", lt["ffn_gate"], E, FF, sigma)
        mat(b + "ffn_down.weight", lt["ffn_down"], FF, E, sigma)
        mat(b + "ffn_up.weight", lt["ffn_up"], E, FF, sigma)
    vec("output_norm.weight", E)
    mat("output.weight", out_t, E, shape.n_vocab, sigma * 2)
    w.write()
    return dict(path=str(path), weight_bytes_per_token=per_token[0], tensor_types=types_used)


def write_falcon(path, shape: FalconShape = FALCON_7B_SHAPED, ftype="Q5_K_M", seed=0, quantizer=None, sigma=0.02, emb_sigma=1.0, token_rows=None,
                 tensor_types=None):
    """Falcon-architecture GGUF (fused attn_qkv, LayerNorm with bias, gpt2/BPE vocabulary); token_rows and tensor_types as for
    write_llama."""
    main, _, _, emb_t = _type_plan(ftype)
    tensor_types = tensor_types or {}
    out_t = Q8_0 if ftype not in ("F16", "F32") else main
    w = GGUFWriter(path)
    a = "falcon"
    w.add_str("general.architecture", a)
    w.add_str("general.name", f"synthetic-{a}-{ftype}")
    w.add_u32(f"{a}.context_length", shape.n_ctx_train)
    w.add_u32(f"{a}.embedding_length", shape.n_embd)
    w.add_u32(f"{a}.block_count", shape.n_layer)
    w.add_u32(f"{a}.feed_forward_length", shape.n_ff)
    w.add_u32(f"{a}.attention.head_count", shape.n_head)
    w.add_u32(f"{a}.attention.head_count_kv", shape.n_head_kv)
    w.add_f32(f"{a}.attention.layer_norm_epsilon", shape.eps)
    toks, scores, types, merges = make_bpe_vocab(shape.n_vocab)
    w.add_str("tokenizer.ggml.model", "gpt2")
    w.add_arr_str("tokenizer.ggml.tokens", toks)
    w.add_arr_f32("tokenizer.ggml.scores", scores)
    w.add_arr_i32("tokenizer.ggml.token_type", types)
    w.add_arr_str("tokenizer.ggml.merges", merges)
    w.add_u32("tokenizer.ggml.bos_token_id", 11)
    w.add_u32("tokenizer.ggml.eos_token_id", 11)

    E, FF = shape.n_embd, shape.n_ff
    hd = E // shape.n_head
    QKV = (shape.n_head + 2 * shape.n_head_kv) * hd
    sid = [seed * 100003 + 7]
    per_token = [0]
    types_used = {}

    def mat(name, t, ne0, rows, sg, count=True):
        sid[0] += 1
        t = tensor_types.get(name.split(".")[-2], t)
        w.add_tensor(name, t, (ne0, rows), _weight_producer(t, ne0, rows, sg, sid[0], quantizer))
        types_used[name] = t
        if count:
            per_token[0] += tensor_nbytes(t, ne0, rows)

    def vec(name, n, base):
        sid[0] += 1
        s = sid[0]
        w.add_tensor(name, F32, (n,), lambda: (base + 0.1 * np.random.default_rng(s).standard_normal(n, dtype=np.float32)).astype(np.float32))

    if token_rows is None:
        mat("token_embd.weight", emb_t, E, shape.n_vocab, emb_sigma, count=False)
    else:
        sid[0] += 1
        w.add_tensor("token_embd.weight", F32, (E, shape.n_vocab), _f32_table(shape.n_vocab, E, emb_sigma, sid[0], token_rows))
        types_used["token_embd.weight"] = F32
    for il in range(shape.n_layer):
        b = f"blk.{il}."
        lt = _layer_types(ftype, True, il, shape.n_layer)
        vec(b + "attn_norm.weight", E, 1.0)
        vec(b + "attn_norm.bias", E, 0.0)
        mat(b + "attn_qkv.weight", lt["attn_qkv"], E, QKV, sigma)
        mat(b + "attn_output.weight", lt["attn_output"], E, E, sigma)
        mat(b + "ffn_up.weight", lt["ffn_up"], E, FF, sigma)
        mat(b + "ffn_down.weight", lt["ffn_down"], FF, E, sigma)
    vec("output_norm.weight", E, 1.0)
    vec("output_norm.bias", E, 0.0)
    mat("output.weight", out_t, E, shape.n_vocab, sigma * 2)
    w.write()
    return dict(path=str(path), weight_bytes_per_token=per_token[0], tensor_types=types_used)


# ------------------------------------------------------------------------------------------------------------------
# GPT-2 in the old GGML ".bin" container (BASELINE.json configs[0]: the reference's own CPU-runnable case; the CUDA library
# does not serve this format — see DESIGN.md §8).  Layout per the reference loader: magic, six int32 hyper-parameters,
# vocabulary (count, then length-prefixed strings), then tensors {n_dims, name length, type, ne[], name, data}
# (reference: models/llms/gpt2.cc:60-250).
@dataclass
class GPT2Shape:
    n_vocab: int = 50257
    n_ctx: int = 1024
    n_embd: int = 768
    n_head: int = 12
    n_layer: int = 12


GPT2_117M = GPT2Shape()


def write_gpt2_ggml(path, shape: GPT2Shape = GPT2_117M, ftype="Q4_0", seed=0, sigma=0.02):
    import struct
    wt = {"Q4_0": Q4_0, "F16": F16, "F32": F32}[ftype]
    file_ftype = {"F32": 0, "F16": 1, "Q4_0": 2}[ftype] + (2000 if ftype == "Q4_0" else 0)   # GGML_QNT_VERSION 2 * 1000 + ftype
    rng = np.random.default_rng(seed)
    E, V, C = shape.n_embd, shape.n_vocab, shape.n_ctx
    assert E % BLOCK[wt][0] == 0

    def tensor(f, name, t, ne):       # ne[0] is the contiguous dimension
        rows = int(np.prod(ne[1:])) if len(ne) > 1 else 1
        if t == F32 and len(ne) == 1:
            data = (np.ones(ne[0], np.float32) if name.endswith("/g") else (rng.standard_normal(ne[0]) * 0.01).astype(np.float32)).view(np.uint8)
        else:
            data = random_blocks(t, ne[0], rows, sigma, rng)
        nm = name.encode()
        f.write(struct.pack("<iii", len(ne), len(nm), t))
        f.write(struct.pack("<" + "i" * len(ne), *ne))
        f.write(nm)
        f.write(np.ascontiguousarray(data).tobytes())

    with open(path, "wb") as f:
        f.write(struct.pack("<I", 0x67676D6C))
        f.write(struct.pack("<iiiiii", V, C, E, shape.n_head, shape.n_layer, file_ftype))
        f.write(struct.pack("<i", V))
        for i in range(V):
            w = (chr(33 + i) if i < 94 else f"<{i}>").encode()
            f.write(struct.pack("<I", len(w)))
            f.write(w)
        tensor(f, "model/ln_f/g", F32, [E]); tensor(f, "model/ln_f/b", F32, [E])
        tensor(f, "model/wte", wt, [E, V]); tensor(f, "model/wpe", F32, [E, C])
        for i in range(shape.n_layer):
            h = f"model/h{i}/"
            tensor(f, h + "ln_1/g", F32, [E]); tensor(f, h + "ln_1/b", F32, [E])
            tensor(f, h + "ln_2/g", F32, [E]); tensor(f, h + "ln_2/b", F32, [E])
            tensor(f, h + "attn/c_attn/w", wt, [E, 3 * E]); tensor(f, h + "attn/c_attn/b", F32, [3 * E])
            tensor(f, h + "attn/c_proj/w", wt, [E, E]); tensor(f, h + "attn/c_proj/b", F32, [E])
            tensor(f, h + "mlp/c_fc/w", wt, [E, 4 * E]); tensor(f, h + "mlp/c_fc/b", F32, [4 * E])
            tensor(f, h + "mlp/c_proj/w", wt, [4 * E, E]); tensor(f, h + "mlp/c_proj/b", F32, [E])
    return path
