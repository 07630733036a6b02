"""The tensor-sharded mode's fused exchange on one GPU (ctb_xchg_mul_mat, csrc/ops_abi.cu): the cases, their inputs, and the
values every rank's phases must produce, composed from oracle pieces the way test_ops_gpu._pf_expected composes a phase.

One call plays rank `me` of a world of W ranks over n_layers layers.  Per layer the program is P_wo (producer: wo's K range on
the rank's attention slice, + the residual on rank 0), C_up (consumer: RMSNorm of the rank-order fp32 sum of the W partial
vectors, into the rank's rows of w1 with the SiLU table and w3), P_down (w2's K range on silu(gate) * up, + C_up's sum on rank
0) and C_qkv (the rank's rows of wq / wk / wv), the head in its place after the last layer.  The peers' partial vectors are
either random, or (own_peers) what the peers compute from their own shards, so that the sums are a real W-rank run's."""
import ctypes as C

import numpy as np

import q3k_refs
import refs
from ctransformers_b200 import synth, tp_plan
from q3k_refs import Q3_K
from refs import Q4_K, Q5_K, Q6_K, ptr

# the matrices of layer l, entry 7·l + i of the call's list; the last layer has the head at entry 4 and nothing after it
MATS = ("attn_output", "ffn_gate", "ffn_up", "ffn_down", "attn_q", "attn_k", "attn_v")
BASES = (0, 0x7FFFFFFF, 0xFFFFFFFF - 2)   # the exchange count of the first launch: 0xFFFFFFFD wraps past 0 inside the program
MIXED = {"attn_q": Q4_K, "attn_k": Q5_K, "attn_v": Q6_K, "attn_output": Q5_K, "ffn_gate": Q6_K, "ffn_up": Q4_K, "ffn_down": Q4_K, "output": Q5_K}

# name: (n_embd, n_head, n_head_kv, n_ff, n_vocab, world, ranks, types: ftype or MIXED, weight source, own_peers)
CASES = {
    "7b-q4km-w2": (4096, 32, 32, 11008, 4112, 2, (0, 1), "Q4_K_M", "random", True),            # Llama-2-7B Q4_K_M, the real mode
    "7b-q4km-w3": (4096, 32, 32, 11008, 4112, 3, (0, 1, 2), "Q4_K_M", "random", True),         # 6/5/5 head groups, 15/14/14 ff blocks
    "13b-q4km-w4": (5120, 40, 40, 13824, 4112, 4, (0, 3), "Q4_K_M", "random", True),
    "7b-q4km-w8": (4096, 32, 32, 11008, 4112, 8, (0, 5, 7), "Q4_K_M", "random", True),         # XC_MAX_WORLD
    "gqa-q5km-w2": (1024, 8, 2, 2816, 2048, 2, (0, 1), "Q5_K_M", "refq", False),               # modelcases llama_gqa_q5km: whole KV groups
    "q3km-w2": (2048, 16, 16, 5632, 1040, 2, (0, 1), "Q3_K_M", "random", False),               # runs k_step<true, false, true>
    "tiny-mixed-w2": (512, 8, 8, 1280, 300, 2, (0, 1), MIXED, "edge", False),                  # hd 64: a few tiles per phase
}
N_LAYERS = 2   # both parity halves used twice


def shard(n_embd, n_head, n_head_kv, n_ff, world, r):
    """{q: wq rows = wo's K range, g: wk / wv rows, f: w1 / w3 rows = w2's K range} of rank r, from tp_plan."""
    s = tp_plan.plan(n_embd, n_head, n_head_kv, n_ff, 1, world)[r]
    hd = n_embd // n_head
    return {"q": s.attn_k, "g": (s.kv_heads[0] * hd, s.kv_heads[1] * hd), "f": s.ff}


def layer_types(types, il, n_layers=N_LAYERS):
    """{matrix name: ggml type} of layer il (the synth ftype's mix, or a fixed dict), "output" included."""
    if isinstance(types, dict):
        return dict(types)
    t = synth._layer_types(types, False, il, n_layers)
    t["output"] = synth._type_plan(types)[2]
    return t


def weights(t, k, m, seed, src):
    """m rows of k type-t weights from source src (random / refq / edge), as test_ops_gpu makes them."""
    if t == Q3_K:
        return np.ascontiguousarray(q3k_refs.blocks(src, k, m, seed))
    if src == "random":
        return np.ascontiguousarray(synth.random_blocks(t, k, m, 0.02, np.random.default_rng(seed))).view(np.uint8)
    return np.ascontiguousarray({"refq": refs.reference_quantized_blocks, "edge": refs.edge_blocks}[src](t, k, m, seed))


def shapes(c, l, n_layers=N_LAYERS):
    """(name, rows, K) of every matrix of layer l in the call's order."""
    E, nh, nkv, F, V = c[:5]
    G = nkv * (E // nh)
    full = {"attn_output": (E, E), "ffn_gate": (F, E), "ffn_up": (F, E), "ffn_down": (E, F), "attn_q": (E, E), "attn_k": (G, E), "attn_v": (G, E)}
    names = MATS if l < n_layers - 1 else MATS[:4] + ("output",)
    return [(n, *(full[n] if n != "output" else (V, E))) for n in names]


def model(c, seed, n_layers=N_LAYERS):
    """(types, mats) of the call: the full matrices of every layer in MATS order, the head last."""
    types, mats = [], []
    for l in range(n_layers):
        lt = layer_types(c[7], l, n_layers)
        for i, (name, m, k) in enumerate(shapes(c, l, n_layers)):
            types.append(lt[name])
            mats.append(weights(lt[name], k, m, seed + 100 * l + i, c[8]))
    return types, mats


def k_slice(t, w, m, k, k0, k1):
    """The blocks [k0, k1) of every row of an m x k matrix of type t, packed."""
    blk, bb = refs.BLOCK[t]
    return np.ascontiguousarray(w.reshape(m, k // blk, bb)[:, k0 // blk:k1 // blk]).reshape(-1)


def row_slice(t, w, k, r0, r1):
    rb = refs.row_bytes(t, k)
    return np.ascontiguousarray(w.reshape(-1, rb)[r0:r1]).reshape(-1)


def mul_mat(t, w, y):
    """orc_mul_mat of the rows w (whole rows of len(y) weights) by y."""
    k = y.size
    m = w.size // refs.row_bytes(t, k)
    v = np.zeros(m, np.float32)
    assert refs.oracle().orc_mul_mat(t, ptr(w), ptr(np.ascontiguousarray(y, np.float32)), ptr(v), k, m, 1) == 0
    return v


def rms_norm(x, w, eps):
    y = np.zeros_like(x)
    refs.oracle().orc_rms_norm_mul(ptr(x), ptr(w), ptr(y), x.size, eps)
    return y


def silu(v):
    a = np.zeros_like(v)
    refs.oracle().orc_silu(ptr(v), ptr(a), v.size)
    return a


def rank_sum(parts, reverse=False):
    """The consumer's input: the fp32 sum of the ranks' partial vectors in rank order (x = part[0] + part[1] + ...)."""
    order = list(range(len(parts)))[::-1] if reverse else range(len(parts))
    s = None
    for r in order:
        s = parts[r].copy() if s is None else s + parts[r]
    return s


def inputs(c, seed, n_layers=N_LAYERS):
    """(attn [n_layers][n_embd] full attention outputs, res0, norm_w [2·n_layers][n_embd], random peer partials [2·n_layers][W][n_embd])."""
    E, W = c[0], c[5]
    rng = np.random.default_rng(seed)
    attn = (rng.standard_normal((n_layers, E)) * 0.5).astype(np.float32)
    res0 = rng.standard_normal(E).astype(np.float32)
    norm_w = (1 + 0.1 * rng.standard_normal((2 * n_layers, E))).astype(np.float32)
    peers = (rng.standard_normal((2 * n_layers, W, E)) * np.array([0.3, 1.0, 5.0, 0.05])[rng.integers(0, 4, (2 * n_layers, W, 1))]).astype(np.float32)
    return attn, res0, norm_w, peers


def expected(c, me, types, mats, attn, res0, norm_w, peers, eps=1e-5, own_peers=None, reverse=False, res_everywhere=False, n_consumers=None,
             n_layers=N_LAYERS):
    """What rank `me` must produce: {"parts": [exchange][rank] partial vectors (every rank's with own_peers, else me's computed and
    the peers' taken from `peers`), "sums": each consumer's summed input, "outs": each consumer's segment outputs side by side}.
    reverse / res_everywhere: the two mistakes the GPU checks must catch (the sum in reverse rank order, the residual added by
    every rank's producer).  n_consumers: stop after that many consumers."""
    E, nh, nkv, F, V, W = c[:6]
    own = c[9] if own_peers is None else own_peers
    sh = [shard(E, nh, nkv, F, W, r) for r in range(W)]
    ranks = range(W) if own else (me,)
    parts, sums, outs = [], [], []
    res = res0
    n_consumers = 2 * n_layers if n_consumers is None else n_consumers
    for l in range(n_layers):
        m0 = 7 * l
        T = lambda i: types[m0 + i]
        ws = lambda i: mats[m0 + i]

        def produce(k, compute):
            p = [peers[k][r].copy() for r in range(W)]
            for r in ranks:
                p[r] = compute(r)
                if r == 0 or res_everywhere:
                    p[r] = p[r] + res
            parts.append(p)
            return rank_sum(p, reverse)

        # P_wo, C_up
        s = produce(2 * l, lambda r: mul_mat(T(0), k_slice(T(0), ws(0), E, E, *sh[r]["q"]), attn[l][slice(*sh[r]["q"])]))
        y = rms_norm(s, norm_w[2 * l], eps)
        gate_up = {r: (silu(mul_mat(T(1), row_slice(T(1), ws(1), E, *sh[r]["f"]), y)), mul_mat(T(2), row_slice(T(2), ws(2), E, *sh[r]["f"]), y)) for r in ranks}
        sums.append(s)
        outs.append(np.concatenate(gate_up[me]))
        if len(sums) == n_consumers:
            break
        res = s
        # P_down, C_qkv or the head
        s = produce(2 * l + 1, lambda r: mul_mat(T(3), k_slice(T(3), ws(3), E, F, *sh[r]["f"]), gate_up[r][0] * gate_up[r][1]))
        y = rms_norm(s, norm_w[2 * l + 1], eps)
        if l < n_layers - 1:
            q, g = sh[me]["q"], sh[me]["g"]
            o = [mul_mat(T(4), row_slice(T(4), ws(4), E, *q), y), mul_mat(T(5), row_slice(T(5), ws(5), E, *g), y), mul_mat(T(6), row_slice(T(6), ws(6), E, *g), y)]
        else:
            o = [mul_mat(T(4), ws(4), y)]
        sums.append(s)
        outs.append(np.concatenate(o))
        if len(sums) == n_consumers:
            break
        res = s
    return {"parts": parts, "sums": sums, "outs": outs}


def split_mantissa(x, W):
    """W float32 vectors whose fp32 sum in rank order is x bit for bit: part r holds the bits [b_r, b_r+1) of each element's 24-bit
    significand (b_r = 24·r / W; rank 0 the low bits, the last rank the high ones), with the element's sign and exponent.  Every
    partial sum is a run of the significand's bits, so no addition rounds.  Zeros and subnormals go whole to the last rank, the
    other ranks holding a zero of the element's sign."""
    x = np.asarray(x, np.float32)
    m, e = np.frexp(x.astype(np.float64))             # x = m · 2^e, 0.5 <= |m| < 1
    sig = np.round(np.abs(m) * 2.0 ** 24).astype(np.int64)
    normal = (x != 0) & (np.abs(x) >= np.finfo(np.float32).tiny)
    bounds = [24 * r // W for r in range(W + 1)]
    parts = []
    for r in range(W):
        bits = sig & (((1 << bounds[r + 1]) - 1) ^ ((1 << bounds[r]) - 1))
        p = (np.sign(m) * np.ldexp(bits.astype(np.float64), e - 24)).astype(np.float32)
        parts.append(np.where(normal, p, np.copysign(np.float32(0), x)))
    parts[-1] = np.where(normal, parts[-1], x)
    return parts


def run(lib, c, me, types, mats, attn, res0, norm_w, peer_parts, base, steps=2, eps=1e-5, n_layers=N_LAYERS, **over):
    """ctb_xchg_mul_mat for rank me; returns (rc, out, sum_out, ll [n_layers][W][2][W][n_embd][2], sync2, launch).  peer_parts:
    [exchange][rank] vectors (me's entries are not passed).  over: argument overrides for the refusal checks."""
    E, nh, nkv, F, V, W = c[:6]
    a = dict(world=W, rank=me, n_embd=E, n_head=nh, n_head_kv=nkv, n_ff=F, n_vocab=V, n_layers=n_layers, steps=steps)
    a.update(over)
    sh = shard(E, nh, nkv, F, W, me) if "world" not in over and "rank" not in over else None
    qw = (sh["q"][1] - sh["q"][0]) if sh else E
    fw = (sh["f"][1] - sh["f"][0]) if sh else F
    gw = (sh["g"][1] - sh["g"][0]) if sh else E
    n_x = 2 * max(n_layers, 1)   # (buffers of one layer at least for the refusal checks)
    att = np.ascontiguousarray(np.stack([attn[l][slice(*sh["q"])] if sh else attn[l] for l in range(max(n_layers, 1))]), np.float32)
    tarr = np.array(types, np.int32)
    wp = (C.c_void_p * len(mats))(*[None if w is None else w.ctypes.data for w in mats])
    keep = [np.ascontiguousarray(peer_parts[k][r], np.float32) if (r != me and peer_parts[k][r] is not None) else None for k in range(n_x) for r in range(W)]
    pp = (C.c_void_p * len(keep))(*[None if v is None else v.ctypes.data for v in keep])
    n_out = sum(2 * fw if k % 2 == 0 else (V if k == n_x - 1 else qw + 2 * gw) for k in range(n_x))
    out = np.full(n_out, np.nan, np.float32)
    sums = np.full((n_x, E), np.nan, np.float32)
    ll = np.full((max(n_layers, 1), W, 2, W, E, 2), 0xDEADBEEF, np.uint32)
    sync2 = np.zeros(1, np.uint32)
    launch = np.full(3, -1, np.int32)
    rc = lib.ctb_xchg_mul_mat(a["world"], a["rank"], a["n_embd"], a["n_head"], a["n_head_kv"], a["n_ff"], a["n_vocab"], a["n_layers"], ptr(tarr),
                              C.cast(wp, C.c_void_p), ptr(att), ptr(res0), ptr(np.ascontiguousarray(norm_w[:n_x])), eps, C.cast(pp, C.c_void_p),
                              base & 0xFFFFFFFF, a["steps"], ptr(out), ptr(sums), ptr(ll), ptr(sync2), ptr(launch))
    return rc, out, sums, ll, int(sync2[0]), tuple(int(v) for v in launch)
