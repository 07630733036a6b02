"""Beam search: the golden cases (tests/golden/beam_search_runs.npz) and a Python restatement of the reference's llama_beam_search
(models/ggml/llama.cpp:4334-4579) driven as its examples/beam_search does (a beam is at its end when its last token is EOS; the
callback collects the common prefix).  The restatement takes an eval function, so it runs on the oracle in the CPU tests, and
its selection step alone checks ctb_beam_step.

Every float that ranks beams follows the reference's order: the row's maximum, a sequential fp32 sum of the host libm's expf(l - max)
in vocabulary order, and the candidates and next beams kept in min-heaps with libstdc++'s make_heap / pop_heap / push_heap, whose
array order decides ties, the renormalising sum and the top beam."""
import ctypes as C
import hashlib

import numpy as np

import logits_all_cases as LA
from ctransformers_b200 import synth

N_PREDICT = 28      # the 37-token prompts then reach position 65: beams' chunks cross the multiple of 32 at 64
BEAM_COUNTS = (1, 2, 4, 8)
MODELS = ("llama_tiny_q4km", "llama_gqa_q5km", "falcon_tiny_q5km", "llama_tiny_q3ks")
BATCH_SIZE = 8      # the prompt's chunking (the config default)

# A small vocabulary whose output rows are scaled up 6x (EOS's 7.8x), so that the distributions are peaked and EOS reaches the beams:
# beams end, and runs stop on an eob top beam before n_predict.
SMALL = "llama_small_vocab"
SMALL_SHAPE = synth.LlamaShape(n_vocab=330, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=1, n_ctx_train=128)
SMALL_CTX = 96
SMALL_SEEDS = tuple(range(6))
SMALL_BEAMS = (2, 4, 8)


def cases():
    """key -> (model name, prompt, n_beams, n_predict)"""
    out = {}
    for name in MODELS:
        for nb in BEAM_COUNTS:
            out[f"{name}_b{nb}"] = (name, LA.prompt(name), nb, N_PREDICT)
    for seed in SMALL_SEEDS:
        for nb in SMALL_BEAMS:
            out[f"{SMALL}_s{seed}_b{nb}"] = (SMALL, small_prompt(seed), nb, N_PREDICT)
    return out


def small_prompt(seed):
    ids = np.random.default_rng(100 + seed).integers(3, SMALL_SHAPE.n_vocab, 40).tolist()
    ids[0] = 1
    return ids


def build(name, directory):
    """(path, n_ctx) of a case's model file"""
    from pathlib import Path
    if name == SMALL:
        path = Path(directory) / f"{SMALL}.gguf"
        if not path.exists():
            synth.write_llama(path, SMALL_SHAPE, "Q4_K_M", seed=0, quantizer=_small_blocks)
        return path, SMALL_CTX
    return LA.build(name, directory)


def _small_blocks(t, w):
    """random blocks (synth.random_blocks, seeded by the drawn matrix); the Q6_K output's row scales 6x, EOS's 7.8x"""
    rng = np.random.default_rng(int.from_bytes(hashlib.sha256(w.tobytes()).digest()[:8], "little"))
    out = synth.random_blocks(t, w.shape[1], w.shape[0], 0.02, rng)
    if t == synth.Q6_K and w.shape[0] == SMALL_SHAPE.n_vocab:
        blk = out.reshape(SMALL_SHAPE.n_vocab, -1)
        d = blk[:, 208:210].copy().view(np.float16)[:, 0].astype(np.float32) * 6
        d[2] *= 1.3
        blk[:, 208:210] = d.astype(np.float16)[:, None].view(np.uint8)
    return out


def eos_of(name):
    return 11 if arch_of(name) == "falcon" else 2


def n_vocab_of(name):
    return SMALL_SHAPE.n_vocab if name == SMALL else LA.n_vocab(name)


def arch_of(name):
    return "llama" if name == SMALL else LA.arch(name)


# ----------------------------------------------------------------------------------------- libstdc++'s heap algorithms
def _push_heap(a, hole, top, value, comp):
    parent = (hole - 1) // 2
    while hole > top and comp(a[parent], value):
        a[hole] = a[parent]
        hole = parent
        parent = (hole - 1) // 2
    a[hole] = value


def _adjust_heap(a, hole, n, value, comp):
    top, child = hole, hole
    while child < (n - 1) // 2:
        child = 2 * (child + 1)
        if comp(a[child], a[child - 1]):
            child -= 1
        a[hole] = a[child]
        hole = child
    if n % 2 == 0 and child == (n - 2) // 2:
        child = 2 * (child + 1)
        a[hole] = a[child - 1]
        hole = child - 1
    _push_heap(a, hole, top, value, comp)


def make_heap(a, comp):
    n = len(a)
    if n < 2:
        return
    parent = (n - 2) // 2
    while True:
        _adjust_heap(a, parent, n, a[parent], comp)
        if parent == 0:
            return
        parent -= 1


def pop_heap(a, comp):
    if len(a) > 1:
        last = len(a) - 1
        value = a[last]
        a[last] = a[0]
        _adjust_heap(a, 0, last, value, comp)


def push_heap(a, comp):
    _push_heap(a, len(a) - 1, 0, a[-1], comp)


# ----------------------------------------------------------------------------------------- the selection step
_libm = None


def expf(x):
    global _libm
    if _libm is None:
        _libm = C.CDLL("libm.so.6")
        _libm.expf.restype, _libm.expf.argtypes = C.c_float, [C.c_float]
    return np.float32(_libm.expf(float(x)))


def f32(x):
    return np.float32(x)


class Beam:
    """tokens: after the prompt, as the reference's beam holds them (its common prefix shifted off); parent / token: where it
    came from in the step before (token -1: an eob beam carried over)."""
    __slots__ = ("tokens", "p", "eob", "parent", "token")

    def __init__(self, tokens, p, eob, parent=-1, token=-1):
        self.tokens, self.p, self.eob, self.parent, self.token = list(tokens), f32(p), bool(eob), parent, token


def top_k(row, k):
    """llama_logit_info::top_k: [(id, logit)] in heap array order"""
    comp = lambda a, b: a[1] > b[1]
    k_min = min(k, len(row))
    heap = [(i, row[i]) for i in range(k_min)]
    make_heap(heap, comp)
    front = heap[0][1]
    for i in np.flatnonzero(row > front) if k_min else []:   # (ids whose logit beats the front at the start; re-tested in order)
        if i < k_min:
            continue
        if heap[0][1] < row[i]:
            pop_heap(heap, comp)
            heap[-1] = (int(i), row[i])
            push_heap(heap, comp)
    return heap


def logit_info(row):
    """(max, normaliser) of llama_logit_info: the first maximum; 1 / sequential fp32 sum of expf(l - max)"""
    m = f32(row.max()) if not np.isnan(row).any() else _first_max(row)
    s = f32(0)
    with np.errstate(over="ignore", invalid="ignore"):   # (inf - inf is NaN and a finite overflow -inf, as in C)
        diff = (row - m).astype(np.float32)
    for v in diff:
        s = f32(s + expf(v))
    return m, f32(f32(1) / s)


def _first_max(row):
    best = row[0]
    for v in row[1:]:
        if best < v:
            best = v
    return f32(best)


class Underflow(Exception):
    pass


def fill(n_beams, beam, parent, row, nxt):
    """fill_next_beams_by_top_probabilities for one beam (children get parent / token)"""
    comp = lambda a, b: a.p > b.p
    if beam.eob:
        carried = Beam(beam.tokens, beam.p, True, parent, -1)
        if len(nxt) < n_beams:
            nxt.append(carried)
            if len(nxt) == n_beams:
                make_heap(nxt, comp)
        elif nxt[0].p < carried.p:
            pop_heap(nxt, comp)
            nxt[-1] = carried
            push_heap(nxt, comp)
        return
    max_l, norm = logit_info(row)
    top = top_k(row, n_beams)

    def child(i):
        tok, logit = top[i]
        with np.errstate(over="ignore", invalid="ignore"):
            return Beam(beam.tokens + [tok], f32(beam.p * f32(norm * expf(f32(logit - max_l)))), False, parent, tok)
    i = 0
    if len(nxt) < n_beams:
        while len(nxt) < n_beams:
            nxt.append(child(i))
            i += 1
        make_heap(nxt, comp)
    else:
        while nxt[0].p == 0:
            if i >= len(top):
                raise Underflow
            pop_heap(nxt, comp)
            nxt[-1] = child(i)
            push_heap(nxt, comp)
            i += 1
    while i < n_beams:
        c = child(i)
        if nxt[0].p < c.p:
            pop_heap(nxt, comp)
            nxt[-1] = c
            push_heap(nxt, comp)
        i += 1


def step(n_beams, beams, nxt, rows):
    """One selection step (ctb_beam_step): nxt (the previous step's beams) zeroed and refilled, then renormalised."""
    for b in nxt:
        b.p, b.parent, b.token = f32(0), -1, -1
    for i, b in enumerate(beams):
        fill(n_beams, b, i, rows[i], nxt)
    if any(b.parent < 0 for b in nxt):
        raise Underflow
    s = f32(0)
    for b in nxt:
        s = f32(s + b.p)
    inv = f32(f32(1) / s)
    for b in nxt:
        b.p = f32(b.p * inv)
    return nxt


def top_index(beams):
    """max_element with llama_beam::operator< on (p, eob): the first maximum"""
    best = 0
    for i in range(1, len(beams)):
        a, b = beams[best], beams[i]
        if (a.p, a.eob) < (b.p, b.eob):
            best = i
    return best


def p_bits(p):
    return int(np.array([p], np.float32).view(np.uint32)[0])


def state_digest(beams, cpl, last_call):
    """SHA-256 of a callback's beam state: n_beams, common prefix length, last_call, then per beam (array order) its token count,
    tokens, p bits and eob flag (after the callback marked it)."""
    words = [len(beams), cpl, int(last_call)]
    for b in beams:
        words += [len(b.tokens), *b.tokens, p_bits(b.p), int(b.eob)]
    return hashlib.sha256(np.array(words, np.int64).tobytes()).hexdigest()


def callback(beams, eos, response, digests, last_call):
    """the example's callback: marks beams ending in EOS, collects the common prefix; returns the common prefix length"""
    cpl = len(beams[0].tokens)
    for b in beams[1:]:
        cpl = min(cpl, len(b.tokens))
        for j in range(cpl):
            if b.tokens[j] != beams[0].tokens[j]:
                cpl = j
                break
    for b in beams:
        if not b.eob and b.tokens and b.tokens[-1] == eos:
            b.eob = True
    response += beams[0].tokens[:cpl]
    digests.append(state_digest(beams, cpl, last_call))
    return cpl


def vp_lanes(p, n_total):
    """whether position p's V·P dots in a chunk of row length n_total add all its elements in the f16 dot's 32 lanes (DESIGN §2,
    item 4): the two sums a position's K / V can come from (ctransformers_b200/csrc/llm_abi.cu vp_lanes)"""
    return (n_total & ~31) >= p + 1


def lane_change(n_past, end):
    """whether a chunk of positions [n_past, end) puts one of them in the other sum than a token-by-token eval"""
    return any(vp_lanes(q, end) != vp_lanes(q, q + 1) for q in range(n_past, end - 1))


def beam_search(eval_fn, n_past, n_beams, n_predict, eos, logits, step_fn=step):
    """llama_beam_search after a prompt of n_past tokens whose last logits row is `logits`.  eval_fn(tokens, n_past) evaluates one
    chunk on the one KV cache and returns its last row; step_fn is the selection step (step's arguments and result).  Returns
    (response, final p, [callback digests], stats) where stats counts the beams' chunk evaluations, and the chunks (common
    prefixes included) that put a position in the other V·P sum than a token-by-token eval would (vp_lanes)."""
    beams, nxt, response, digests = [Beam([], 1.0, False)], [], [], []
    stats = {"evals": 0, "lane_changes": 0}
    i = 0
    while i < n_predict and any(not b.eob for b in beams) and not beams[top_index(beams)].eob:
        cpl = callback(beams, eos, response, digests, False)
        if cpl:
            logits = eval_fn(beams[0].tokens[:cpl], n_past)
            stats["lane_changes"] += lane_change(n_past, n_past + cpl)
            n_past += cpl
        rows = []
        for b in beams:
            b.tokens = b.tokens[cpl:]
            if b.eob:
                rows.append(None)
                continue
            if b.tokens:
                logits = eval_fn(b.tokens, n_past)
                stats["evals"] += 1
                stats["lane_changes"] += lane_change(n_past, n_past + len(b.tokens))
            rows.append(np.array(logits, np.float32))
        new = step_fn(n_beams, beams, nxt, rows)
        nxt, beams = beams, new
        i += 1
    t = top_index(beams)
    beams = [beams[t]]
    callback(beams, eos, response, digests, True)
    return response, beams[0].p, digests, stats
