"""ctypes loaders for the two CHECKERS (test infrastructure, never the product):

  * ``oracle()``  — oracle/_build/liboracle.so, our plain-C restatement (oracle/ggml_oracle.c)
  * ``ref()``     — oracle/_ref/libctransformers_ref.so, the unmodified reference compiled by oracle/Makefile where its
                    sources are available; only tests/golden/make_golden.py uses it.  The tests compare with what it
                    computed, stored under tests/golden/.
"""
import ctypes as C
import hashlib
import os
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE_SO = ROOT / "oracle" / "_build" / "liboracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libctransformers_ref.so"

# ggml type ids (ggml.h enum ggml_type)
F32, F16, Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K, Q8_K = 0, 1, 2, 6, 8, 12, 13, 14, 15
BLOCK = {Q4_0: (32, 18), Q5_0: (32, 22), Q8_0: (32, 34), Q4_K: (256, 144), Q5_K: (256, 176), Q6_K: (256, 210), Q8_K: (256, 292),
         F32: (1, 4), F16: (1, 2)}
TYPE_NAME = {Q4_0: "q4_0", Q5_0: "q5_0", Q8_0: "q8_0", Q4_K: "q4_K", Q5_K: "q5_K", Q6_K: "q6_K"}


def row_bytes(t, k):
    bs, sz = BLOCK[t]
    assert k % bs == 0
    return k // bs * sz


_oracle = None
_ref = None


def oracle():
    global _oracle
    if _oracle is None:
        if not ORACLE_SO.exists():
            subprocess.check_call(["make", "-C", str(ROOT / "oracle"), "oracle"])
        o = C.CDLL(str(ORACLE_SO))
        fp, vp, i = C.POINTER(C.c_float), C.c_void_p, C.c_int
        o.orc_fp16_to_fp32.restype = C.c_float
        o.orc_fp16_to_fp32.argtypes = [C.c_uint16]
        o.orc_fp32_to_fp16.restype = C.c_uint16
        o.orc_fp32_to_fp16.argtypes = [C.c_float]
        for n in ("orc_vec_dot_q4_0_q8_0", "orc_vec_dot_q5_0_q8_0", "orc_vec_dot_q8_0_q8_0", "orc_vec_dot_q4_K_q8_K", "orc_vec_dot_q5_K_q8_K",
                  "orc_vec_dot_q6_K_q8_K"):
            getattr(o, n).restype = C.c_float
            getattr(o, n).argtypes = [i, vp, vp]
        o.orc_mul_mat.restype = i
        o.orc_mul_mat.argtypes = [i, vp, vp, vp, i, i, i]
        o.orc_rms_norm_mul.argtypes = [vp, vp, vp, i, C.c_float]
        o.orc_layer_norm_mul_add.argtypes = [vp, vp, vp, vp, i, C.c_float]
        o.orc_rope.argtypes = [vp, i, i, i, i, C.c_float, C.c_float]
        o.orc_rope_table.argtypes = [vp, i, i, C.c_float, C.c_float]
        o.orc_attn_head.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, i, i, C.c_float, vp]
        _oracle = o
    return _oracle


class _Traits(C.Structure):
    _fields_ = [("type_name", C.c_char_p), ("blck_size", C.c_int), ("type_size", C.c_size_t), ("is_quantized", C.c_bool),
                ("to_float", C.c_void_p), ("from_float", C.c_void_p), ("from_float_reference", C.c_void_p),
                ("vec_dot", C.c_void_p), ("vec_dot_type", C.c_int)]


def have_ref():
    return REF_SO.exists()


def ref():
    """The compiled reference (AVX2 build).  Also initialises ggml's fp16 tables once."""
    global _ref
    if _ref is None:
        r = C.CDLL(str(REF_SO))
        r.ggml_internal_get_type_traits.restype = _Traits
        r.ggml_internal_get_type_traits.argtypes = [C.c_int]

        class _IP(C.Structure):
            _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]
        r.ggml_init.restype = C.c_void_p
        r.ggml_init.argtypes = [_IP]
        r.ggml_free.argtypes = [C.c_void_p]
        r.ggml_free(r.ggml_init(_IP(1 << 20, None, False)))  # builds table_silu_f16 & co (ggml.c:4319-4333)
        r.ggml_quantize_chunk.restype = C.c_size_t
        r.ggml_quantize_chunk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        _ref = r
    return _ref


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


GOLD = ROOT / "tests" / "golden"


def golden_runs():
    """What the reference computed for the tests that compare with it (tests/golden/make_golden.py reference_runs)."""
    return np.load(GOLD / "reference_runs.npz")


def digest(a):
    """SHA-256 of an array's bytes (float32 vectors, quantized blocks): a bit-exact stand-in for a stored vector."""
    a = np.ascontiguousarray(a)
    assert a.dtype in (np.float32, np.uint8), a.dtype
    return hashlib.sha256(a.tobytes()).hexdigest()


def reference_quantized_blocks(t, k, m, seed):
    """m rows of k weights of type t (bytes), assembled from blocks the reference's quantizer produced (reference_blocks.npz:
    256 K-quant or 1024 32-weight blocks per type).  Each block is quantized on its own, so any arrangement of them is a
    matrix the reference's quantizer could have written, with the scale / min bit patterns that random blocks do not reach."""
    bs, sz = BLOCK[t]
    pool = np.load(GOLD / "reference_blocks.npz")[f"blocks_{t}"]
    idx = np.random.default_rng(seed).integers(0, len(pool), m * (k // bs))
    return np.ascontiguousarray(pool[idx].reshape(-1))


def _f16_edge(rng, n):
    """n f16 bit patterns of both signs: mostly normal values 2^-16 .. 2^-6, a fifth subnormal (bits 1 .. 1023), a few zeros."""
    mag = np.exp2(rng.uniform(-16, -6, n)).astype(np.float16).view(np.uint16)
    kind = rng.integers(0, 10, n)
    mag[kind < 2] = rng.integers(1, 1024, int((kind < 2).sum()))
    mag[kind == 9] = 0
    return mag | (rng.integers(0, 2, n).astype(np.uint16) << 15)


def edge_blocks(t, k, m, seed):
    """m rows of k weights of type t (Q4_K / Q5_K / Q6_K bytes) at the edges of the block formats, where random_blocks and the
    reference's quantizer do not go.  Sub-block scales and mins are drawn from shuffled runs of all their values, independently
    of each other: blocks 8i .. 8i+7 together hold every 6-bit scale and every 6-bit min (Q4_K / Q5_K), blocks 16i .. 16i+15
    every Q6_K scale -128..127.  Whole sub-blocks have all-zero or all-set quants (and for Q5_K / Q6_K only the low or only the high bits set),
    d and dmin have both signs and reach f16 subnormals and zero; no inf or NaN."""
    rng = np.random.default_rng(seed)
    bs, sz = BLOCK[t]
    nb = m * (k // bs)
    nsub, qmax, consts = {Q4_K: (8, 15, (0, 15)), Q5_K: (8, 31, (0, 31, 15, 16)), Q6_K: (16, 63, (0, 63, 15, 48))}[t]

    def runs(values, n):   # n draws: concatenated shuffles of all values
        return np.concatenate([rng.permutation(values) for _ in range(-(-n // len(values)))])[:n].reshape(nb, -1)

    q = rng.integers(0, qmax + 1, (nb, nsub, 256 // nsub))
    pat = np.arange(nb * nsub).reshape(nb, nsub) % (2 * len(consts))   # every other sub-block random, the rest cycle the constants
    for i, c in enumerate(consts):
        q[pat == 2 * i + 1] = c
    q = q.reshape(nb, 256)
    out = np.zeros((nb, sz), np.uint8)
    if t in (Q4_K, Q5_K):
        sc, mn = runs(np.arange(64), nb * 8), runs(np.arange(64), nb * 8)
        out[:, 0:2] = _f16_edge(rng, nb).view(np.uint8).reshape(nb, 2)
        out[:, 2:4] = _f16_edge(rng, nb).view(np.uint8).reshape(nb, 2)
        s = out[:, 4:16]                                                  # inverse of get_scale_min_k4 (k_quants.c:306-313)
        s[:, 0:4] = sc[:, 0:4] | ((sc[:, 4:8] >> 4) << 6)
        s[:, 4:8] = mn[:, 0:4] | ((mn[:, 4:8] >> 4) << 6)
        s[:, 8:12] = (sc[:, 4:8] & 0xF) | ((mn[:, 4:8] & 0xF) << 4)
        qs = out[:, 16:144] if t == Q4_K else out[:, 48:176]
        for j in range(4):                                                # 64 weights per 32 bytes: sub-block 2j low nibbles, 2j+1 high
            lo, hi = q[:, 64 * j:64 * j + 32], q[:, 64 * j + 32:64 * j + 64]
            qs[:, 32 * j:32 * j + 32] = (lo & 15) | ((hi & 15) << 4)
            if t == Q5_K:                                                 # qh bit 2j / 2j+1 of byte l: 5th bit of weight l of those sub-blocks
                out[:, 16:48] |= ((lo >> 4) << (2 * j) | (hi >> 4) << (2 * j + 1)).astype(np.uint8)
    else:   # Q6_K: ql[128] qh[64] scales[16] d (dequantize_row_q6_K, k_quants.c:1083-1117)
        out[:, 192:208] = runs(np.arange(-128, 128), nb * 16).astype(np.int8).view(np.uint8)
        out[:, 208:210] = _f16_edge(rng, nb).view(np.uint8).reshape(nb, 2)
        for n in range(2):
            for j in range(4):
                v = q[:, 128 * n + 32 * j:128 * n + 32 * j + 32]
                out[:, 64 * n + 32 * (j & 1):64 * n + 32 * (j & 1) + 32] |= ((v & 15) << (4 * (j >> 1))).astype(np.uint8)
                out[:, 128 + 32 * n:128 + 32 * n + 32] |= ((v >> 4) << (2 * j)).astype(np.uint8)
    return np.ascontiguousarray(out.reshape(-1))


def ref_traits(t):
    tr = ref().ggml_internal_get_type_traits(t)
    to_float = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int)(tr.to_float) if tr.to_float else None
    from_float = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int)(tr.from_float) if tr.from_float else None
    vec_dot = C.CFUNCTYPE(None, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p)(tr.vec_dot) if tr.vec_dot else None
    return dict(to_float=to_float, from_float=from_float, vec_dot=vec_dot, vec_dot_type=tr.vec_dot_type)


def ref_quantize(t, x):
    """Quantize f32 rows [M,K] with the reference's own quantizer (ggml.c:19319 ggml_quantize_chunk)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    m, k = x.shape
    out = np.zeros(m * row_bytes(t, k), dtype=np.uint8)
    hist = np.zeros(16, dtype=np.int64)
    n = ref().ggml_quantize_chunk(t, ptr(x), ptr(out), 0, m * k, ptr(hist))
    assert n == out.size, (n, out.size)
    return out


def ref_quantize_act(t, x):
    """Quantize an activation row with the reference's from_float for type t (Q8_K / Q8_0)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros(row_bytes(t, x.size), dtype=np.uint8)
    ref_traits(t)["from_float"](ptr(x), ptr(out), x.size)
    return out


def ref_vec_dot(t, k, wrow, act):
    s = np.zeros(1, dtype=np.float32)
    ref_traits(t)["vec_dot"](k, ptr(s), ptr(wrow), ptr(act))
    return float(s[0])


def attention_expected(q, k_new, v_new, kcache, vcache, n_head, n_kv, hd, pos0, n_total, mode, freq_base, kq_scale):
    """What the reference's attention block computes for an eval chunk of n_tok tokens at positions pos0.. (llama.cpp:2303-2400),
    from oracle pieces: orc_rope on q and k, the chunk's K rows and V columns stored as fp16 before any token attends, then
    orc_attn_head_n per head over the chunk row length n_total[i].  Arguments as ctb_attention_path (kcache [n_ctx][n_kv*hd],
    vcache [n_kv*hd][n_ctx], uint16 fp16 bits); returns (out [n_tok][n_head*hd], kcache, vcache) with the new rows stored."""
    o = oracle()
    o.orc_attn_head_n.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]
    n_tok, n_ctx = q.shape[0], kcache.shape[0]
    kc, vc = kcache.copy(), vcache.copy()
    for i in range(n_tok):
        kr = np.ascontiguousarray(k_new[i], np.float32).copy()
        o.orc_rope(ptr(kr), n_kv, hd, pos0 + i, mode, freq_base, 1.0)
        kc[pos0 + i] = kr.astype(np.float16).view(np.uint16)
        vc[:, pos0 + i] = np.asarray(v_new[i], np.float32).astype(np.float16).view(np.uint16)
    out = np.zeros((n_tok, n_head * hd), np.float32)
    group = n_head // n_kv
    for i in range(n_tok):
        T = pos0 + i + 1
        assert T <= n_total[i] <= n_ctx
        qr = np.ascontiguousarray(q[i], np.float32).copy()
        o.orc_rope(ptr(qr), n_head, hd, pos0 + i, mode, freq_base, 1.0)
        for h in range(n_head):
            kvh = h // group
            o.orc_attn_head_n(ptr(qr[h * hd:]), kc.ctypes.data + kvh * hd * 2, n_kv * hd, vc.ctypes.data + kvh * hd * n_ctx * 2, n_ctx, hd, T,
                              int(n_total[i]), float(kq_scale), out.ctypes.data + (i * n_head + h) * hd * 4)
    return out, kc, vc


# --------------------------------------------------------------------------------------------------------------
# Whole-model oracle (oracle/llama_oracle.c) driven from a GGUF file
def read_gguf(path):
    """Tiny GGUF v2/v3 reader: returns (kv dict, {name: (type, shape, np.uint8 view of the data)})."""
    import struct
    buf = np.memmap(path, dtype=np.uint8, mode="r")
    pos = [0]

    def rd(fmt):
        v = struct.unpack_from("<" + fmt, buf, pos[0])
        pos[0] += struct.calcsize("<" + fmt)
        return v[0] if len(v) == 1 else v

    def rstr():
        n = rd("Q")
        s = bytes(buf[pos[0]:pos[0] + n])
        pos[0] += n
        return s

    scalar = {0: "B", 1: "b", 2: "H", 3: "h", 4: "I", 5: "i", 6: "f", 7: "?", 10: "Q", 11: "q", 12: "d"}
    magic, version, n_tensors, n_kv = rd("I"), rd("I"), rd("Q"), rd("Q")
    assert magic == 0x46554747 and version >= 2
    kv = {}
    for _ in range(n_kv):
        key = rstr().decode()
        t = rd("I")
        if t == 8:
            kv[key] = rstr()
        elif t == 9:
            et, n = rd("I"), rd("Q")
            if et == 8:
                kv[key] = [rstr() for _ in range(n)]
            else:
                sz = struct.calcsize(scalar[et])
                kv[key] = np.frombuffer(buf, dtype=np.dtype("<" + scalar[et]), count=n, offset=pos[0]).copy()
                pos[0] += sz * n
        else:
            kv[key] = rd(scalar[t])
    infos = []
    for _ in range(n_tensors):
        name = rstr().decode()
        nd = rd("I")
        shape = [rd("Q") for _ in range(nd)]
        t, off = rd("I"), rd("Q")
        infos.append((name, t, shape, off))
    align = kv.get("general.alignment", 32)
    start = (pos[0] + align - 1) // align * align
    tensors = {}
    for name, t, shape, off in infos:
        rows = int(np.prod(shape[1:])) if len(shape) > 1 else 1
        nbytes = row_bytes(t, shape[0]) * rows
        tensors[name] = (t, shape, buf[start + off:start + off + nbytes])
    return kv, tensors


class OracleModel:
    """oracle/llama_oracle.c bound to one GGUF file (keeps the arrays alive)."""

    def __init__(self, path, n_ctx):
        o = oracle()
        kv, tensors = read_gguf(path)
        arch = kv["general.architecture"].decode()
        g = lambda k, d=None: kv.get(f"{arch}.{k}", d)
        self.falcon = arch == "falcon"
        self.n_vocab = len(kv["tokenizer.ggml.tokens"])
        self.n_embd, self.n_ff, self.n_head, self.n_layer = g("embedding_length"), g("feed_forward_length"), g("attention.head_count"), g("block_count")
        self.n_head_kv = g("attention.head_count_kv", self.n_head)
        eps = g("attention.layer_norm_epsilon") if self.falcon else g("attention.layer_norm_rms_epsilon")
        rope_base = g("rope.freq_base", 10000.0)
        lin = g("rope.scale_linear", 1.0)
        o.orc_model_new.restype = C.c_void_p
        o.orc_model_new.argtypes = [C.c_int] * 8 + [C.c_float] * 3
        o.orc_model_set_mat.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        o.orc_model_set_vec.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        o.orc_model_set_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        o.orc_model_free.argtypes = [C.c_void_p]
        o.orc_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        self.o, self.keep = o, []
        self.m = o.orc_model_new(int(self.falcon), self.n_vocab, self.n_embd, self.n_ff, self.n_head, self.n_head_kv, self.n_layer, n_ctx,
                                 eps, rope_base, 1.0 / lin if lin != 1.0 else 1.0)

        def mat(layer, slot, name):
            t, shape, data = tensors[name]
            a = np.ascontiguousarray(data)
            self.keep.append(a)
            o.orc_model_set_mat(self.m, layer, slot, t, shape[0], int(np.prod(shape[1:])), ptr(a))

        def vec(layer, slot, name):
            if name not in tensors:
                return
            a = np.ascontiguousarray(tensors[name][2]).view(np.float32)
            self.keep.append(a)
            o.orc_model_set_vec(self.m, layer, slot, ptr(a))

        mat(-1, 0, "token_embd.weight")
        mat(-1, 1, "output.weight")
        vec(-1, 0, "output_norm.weight")
        vec(-1, 1, "output_norm.bias")
        for il in range(self.n_layer):
            b = f"blk.{il}."
            vec(il, 0, b + "attn_norm.weight"); vec(il, 1, b + "attn_norm.bias")
            vec(il, 2, b + "attn_norm_2.weight"); vec(il, 3, b + "attn_norm_2.bias"); vec(il, 4, b + "ffn_norm.weight")
            names = ({3: "attn_qkv", 4: "attn_output", 6: "ffn_down", 7: "ffn_up"} if self.falcon else
                     {0: "attn_q", 1: "attn_k", 2: "attn_v", 4: "attn_output", 5: "ffn_gate", 6: "ffn_down", 7: "ffn_up"})
            for slot, nm in names.items():
                mat(il, slot, b + nm + ".weight")
        self.logits = np.zeros(self.n_vocab, np.float32)
        self.embd = np.zeros(self.n_embd, np.float32)
        self.trace_layers = np.zeros((self.n_layer, self.n_embd), np.float32)
        self.trace_attn = np.zeros((self.n_layer, self.n_embd), np.float32)
        o.orc_model_set_trace(self.m, ptr(self.trace_layers), ptr(self.trace_attn))
        self.n_past = 0

    def set_tp(self, world):
        """Switch the restatement to the sharded engine's summation order (oracle/llama_oracle.c: tp_world)."""
        from ctransformers_b200 import tp_plan
        sh = tp_plan.plan(self.n_embd, self.n_head, self.n_head_kv, self.n_ff, self.n_vocab, world)
        wo = (C.c_int * (world + 1))(*([s.attn_k[0] for s in sh] + [sh[-1].attn_k[1]]))
        w2 = (C.c_int * (world + 1))(*([s.ff[0] for s in sh] + [sh[-1].ff[1]]))
        self.o.orc_model_set_tp.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        assert self.o.orc_model_set_tp(self.m, world, wo, w2) == 0

    def eval(self, tokens, batch_size=8):
        """Same chunking as the reference's LLM::BatchEval (llm.h:40-54): the chunk an attention row belongs to fixes its length."""
        toks = np.asarray(tokens, dtype=np.int32)
        for start in range(0, len(toks), batch_size):
            t = np.ascontiguousarray(toks[start:start + batch_size])
            rc = self.o.orc_eval(self.m, ptr(t), len(t), self.n_past, ptr(self.logits), ptr(self.embd))
            assert rc == 0, rc
            self.n_past += len(t)
        return self.logits

    def __del__(self):
        if getattr(self, "m", None):
            self.o.orc_model_free(self.m)
            self.m = None


# --------------------------------------------------------------------------------------------------------------
# The order of the norms' fp64 sums (csrc/matvec.cuh stage_activation / norm_stat).  The reference adds the terms one after
# another; the kernels' threads add them in chains, a warp butterfly and warp order.  Rows whose terms span many binary orders
# of magnitude round the float statistic differently in the two orders; norm_order_rows plants such rows.
def seq_sum(terms):
    """The reference's order: terms[..., 0] + terms[..., 1] + ... in double (np.cumsum adds in sequence; np.sum is pairwise)."""
    return np.cumsum(np.asarray(terms, np.float64), axis=-1)[..., -1]


def kernel_order_sum(terms, nt):
    """The parallel order of stage_activation + block_sum_f64 with nt threads: thread t adds, starting from 0.0, elements
    (ps*nt + t)*16 .. +15 of every pass ps in pass-major order; the warp butterfly adds the lane sums with xor offsets 16, 8,
    4, 2, 1; the warp sums are then added from 0.0 in warp order."""
    t = np.asarray(terms, np.float64)
    rows = t.reshape(-1, t.shape[-1])
    R, K = rows.shape
    passes = -(-K // (nt * 16))
    pad = np.zeros((R, passes * nt * 16))
    pad[:, :K] = rows
    per = pad.reshape(R, passes, nt, 16).transpose(0, 2, 1, 3).reshape(R, nt, passes * 16)
    lane = np.cumsum(per, axis=-1)[..., -1].reshape(R, nt // 32, 32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[..., idx ^ o]
    return np.cumsum(lane[..., 0], axis=-1)[..., -1].reshape(t.shape[:-1])


def norm_emulated(mode, x, w, b, eps, summer):
    """RMSNorm * w (mode 1) or LayerNorm * w + b (mode 2) of rows x in float32, as orc_rms_norm_mul / orc_layer_norm_mul_add
    compute them, with summer(terms) adding the fp64 sums.  Returns (y, the float statistics: (mean of squares,) or (mean, var))."""
    x = np.atleast_2d(np.asarray(x, np.float32))
    K = x.shape[-1]
    stat = lambda t: (summer(t.astype(np.float64)) / K).astype(np.float32)[:, None]
    f32 = np.float32
    if mode == 1:
        m = stat(x * x)
        scale = f32(1) / np.sqrt(m + f32(eps))
        return (x * scale) * w, (m,)
    mean = stat(x)
    d = x - mean
    var = stat(d * d)
    scale = f32(1) / np.sqrt(var + f32(eps))
    return ((d * scale) * w) + b, (mean, var)


NORM_ORDER_THREADS = tuple(range(64, 1025, 32))   # every CTA size a build can give the kernels (k_step 320, k_pstep 256, k_matvec 512)
NORM_ORDER_EPS = 1e-5


def _planted_row(kind, K, where, rng):
    """One row that breaks the statistic `kind` ("rms": Σx², "mean": Σx, "var": Σ(x - mean)²) in the kernel orders, or None.
    A cluster of large elements carries the sum: x1 and x2 tune it to just below a float rounding boundary of sum / K, and x0
    comes last.  The reference's order then drops every small term after x0 (each is less than half an ulp of the running sum)
    and rounds down; the kernels add the small terms to each other first, keep them and round up.  For "var" every value comes
    with its negation right after it (x0's, the chain of 16 elements it starts holds nothing else), so Σx is exactly 0 in any of
    these orders, the mean is 0 and only Σx² breaks."""
    c = {"start": 0, "middle": K // 2 + 16 * int(rng.integers(0, 8)) + 5, "warp": 509 if K >= 1024 else 13, "end": K - 99}[where]
    sq, var = kind != "mean", kind == "var"
    if var:
        c -= 2                                                     # x0 stays at the same place: the last of its thread's chain
    x = np.zeros(K, np.float32)
    cl = [c, c + 1, c + 2, c + 3, c + 4, c + 5] if var else [c, c + 1, c + 2]
    e_small = float(rng.choice([-27.0, -27.5, -28.0])) if sq else float(rng.choice([-54.0, -55.0, -56.0]))
    small = (np.exp2(e_small) * rng.uniform(0.75, 1.0, K)).astype(np.float32)   # squares (or values) below 2^-54 · x0^2 (x0)
    if var:
        taken = np.zeros(K, bool)
        taken[cl] = True
        xz = cl[-1]
        taken[xz:(xz // 16 + 1) * 16] = True                       # nothing after -x0 in its chain
        for j in range(0, K - 1, 2):
            if not taken[j] and not taken[j + 1]:
                x[j], x[j + 1] = small[j], -small[j]
    else:
        x[:] = small * (rng.choice([-1, 1], K).astype(np.float32) if kind == "rms" else 1)
        x[cl] = 0
    x0 = np.float32(2 + rng.integers(0, 2048) / 1024.0) if not sq else np.float32(1.5 + rng.integers(0, 1024) / 2048.0)
    i0 = cl[-2] if var else cl[-1]
    x[i0] = x0
    if var:
        x[cl[-1]] = -x0

    def terms(r):
        return (r * r).astype(np.float64) if sq else r.astype(np.float64)

    s = seq_sum(terms(x))
    m = np.float32(s / K)
    M = (np.float64(m) + np.float64(np.nextafter(m, np.float32(np.inf)))) / 2   # the rounding boundary above m
    r = M * K - s - 2 * np.spacing(s)                              # what x1 and x2 add, a little short of the boundary
    if var:
        r /= 2
    if r <= 0:
        return None
    f = (lambda v: float(np.float32(v) * np.float32(v))) if sq else float
    parts = []
    for _ in range(2):
        v = np.float32(np.sqrt(r) if sq else r)
        while v > 0 and f(v) > r:
            v = np.nextafter(v, np.float32(0))
        parts.append(v)
        r -= f(v)
    if var:
        x[cl[0]], x[cl[1]], x[cl[2]], x[cl[3]] = parts[0], -parts[0], parts[1], -parts[1]
    else:
        x[cl[0]], x[cl[1]] = parts
    p2 = np.float32(2.0 ** int(np.ceil(np.log2(np.sqrt(K)) if sq else np.log2(K))))   # statistic of order 1: eps does not absorb it
    return x * p2


def _order_breaks(mode, x, w, b):
    """True when, for every thread count in NORM_ORDER_THREADS, the kernel order changes the float statistics and y."""
    want, stats = norm_emulated(mode, x, w, b, NORM_ORDER_EPS, seq_sum)
    for nt in NORM_ORDER_THREADS:
        got, kstats = norm_emulated(mode, x, w, b, NORM_ORDER_EPS, lambda t: kernel_order_sum(t, nt))
        if all(np.array_equal(a, c) for a, c in zip(stats, kstats)) or np.array_equal(got.view(np.uint32), want.view(np.uint32)):
            return False
    return True


def norm_order_rows(mode, K, seed):
    """Planted rows of width K for norm mode 1 (RMSNorm: rows that break Σx²) or 2 (LayerNorm: rows that break Σx, and rows that
    break only Σ(x - mean)²), with the norm weight w and bias b they were checked with.  The cluster of large elements sits at the
    start, in the middle, across a warp boundary (a thread boundary when K < 1024) and near the end; the small terms' size varies
    with the seed.  Every row is checked (_order_breaks) to change the float statistic and y at every thread count."""
    rng = np.random.default_rng(seed)
    w = (1 + 0.1 * rng.standard_normal(K)).astype(np.float32)
    b = (0.1 * rng.standard_normal(K)).astype(np.float32)
    rows = []
    for kind in (("rms",) if mode == 1 else ("mean", "var")):
        for where in ("start", "middle", "warp", "end"):
            for _ in range(64):
                x = _planted_row(kind, K, where, rng)
                if x is not None and _order_breaks(mode, x, w, b):
                    rows.append(x)
                    break
            else:
                raise AssertionError(f"no {kind} row at {where} for K {K}")
    return np.stack(rows), w, b
