"""Beam search on the GPU (MultiLLM.beam_search / beam_search_many, include/ctransformers_b200.h ctb_multi_beam_search): every
response and final p is bit-identical to the reference's llama_beam_search (tests/golden/beam_search_runs.npz), one search at a
time and many sharing launches; the selection step equals the restatement on constructed rows; the re-parenting launch leaves
each beam's K / V byte-equal to a fresh slot's and moves only the positions past the beams' common prefix."""
import ctypes as C

import numpy as np
import pytest

import beam_search_cases as B
import modelcases
import refs
from test_multi_seq_gpu import multi, multi_state, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("beam_gpu_models")


def golden():
    return np.load(refs.GOLD / "beam_search_runs.npz")


def check(key, response, p):
    gold = golden()
    assert response == gold[f"{key}_response"].tolist(), key
    assert B.p_bits(p) == int(gold[f"{key}_p"][0]), (key, p)


_handles = {}


def handle(name, model_dir, n_slots):
    if (name, n_slots) not in _handles:
        path, ctx = B.build(name, model_dir)
        _handles[(name, n_slots)] = multi(path, ctx, n_slots)
    return _handles[(name, n_slots)]


# ------------------------------------------------------------------------------------------ 1. the reference's results
@pytest.mark.parametrize("key", list(B.cases()))
def test_beam_search_matches_reference(key, model_dir):
    name, prompt, nb, n_predict = B.cases()[key]
    m = handle(name, model_dir, 8)
    response, p = m.beam_search(prompt, nb, n_predict, batch_size=B.BATCH_SIZE)
    check(key, response, p)


@pytest.mark.parametrize("name", B.MODELS)
def test_beam_search_many_shares_launches(name, model_dir):
    """A 12-slot handle runs the case's prompt at 4 beams three times over and at 8 beams twice over: the 4-beam searches share
    every launch; the 8-beam ones wait for slots.  Each result is the reference's."""
    m = handle(name, model_dir, 12)
    prompt = B.cases()[f"{name}_b4"][1]
    for nb, copies in ((4, 3), (8, 2)):
        launches = m.launches()
        results = m.beam_search_many([prompt] * copies, nb, B.N_PREDICT, batch_size=B.BATCH_SIZE)
        for response, p in results:
            check(f"{name}_b{nb}", response, p)
        if nb == 4:   # one search alone takes at least one launch per step
            st = m.beam_stats()
            assert 0 < st["steps"] <= B.N_PREDICT + 1 and st["reparent_bytes"] > 0, st
            assert m.launches() - launches < 2 * st["steps"], "the three searches did not share their launches"


def test_small_vocabulary_prompts_together(model_dir):
    """The small-vocabulary prompts, whose beams reach EOS, all in one call: at 4 beams the six searches run at once in 24 of 32
    slots and end at different steps; at 8 beams four run at once and the last two are admitted as slots free up."""
    m = handle(B.SMALL, model_dir, 32)
    prompts = [B.small_prompt(s) for s in B.SMALL_SEEDS]
    for nb in (4, 8):
        results = m.beam_search_many(prompts, nb, B.N_PREDICT, batch_size=B.BATCH_SIZE)
        for s, (response, p) in zip(B.SMALL_SEEDS, results):
            check(f"{B.SMALL}_s{s}_b{nb}", response, p)


@pytest.mark.parametrize("key", ["llama_tiny_q4km_b2", "llama_tiny_q4km_b8", "llama_tiny_q3ks_b8"])
def test_positions_are_evaluated_again_where_the_chunk_changes_their_sum(key, model_dir):
    """Each step evaluates every live beam's newest token, and again the positions whose V·P sum the reference's chunks change
    (beam_search_cases.vp_lanes): one token per beam evaluation when no chunk of the reference's run changes a sum (the first
    case), more when some does (the others)."""
    from test_beam_search import oracle_search
    name, prompt, nb, n_predict = B.cases()[key]
    _, _, _, ref = oracle_search(name, prompt, nb, n_predict, model_dir)
    m = handle(name, model_dir, 8)
    check(key, *m.beam_search(prompt, nb, n_predict, batch_size=B.BATCH_SIZE))
    tokens = m.beam_stats()["tokens"]
    if ref["lane_changes"]:
        assert tokens > len(prompt) + ref["evals"], (tokens, ref)
    else:
        assert tokens == len(prompt) + ref["evals"], (tokens, ref)


# ------------------------------------------------------------------------------------------ 2. the selection step
def beam_step_c(lib, nb, p, eob, rows, n_next):
    n_in, nv = len(p), rows.shape[1]
    rows = np.ascontiguousarray(rows, np.float32)
    op, ot, opp, oe = (C.c_int * nb)(), (C.c_int * nb)(), (C.c_float * nb)(), (C.c_ubyte * nb)()
    r = lib.ctb_beam_step(nb, n_in, n_next, (C.c_float * n_in)(*p), C.cast((C.c_ubyte * n_in)(*eob), C.c_void_p),
                          rows.ctypes.data_as(C.POINTER(C.c_float)), nv, op, ot, opp, C.cast(oe, C.c_void_p))
    return r, [(op[i], ot[i], B.p_bits(opp[i]), oe[i]) for i in range(max(r, 0))]


def beam_step_py(nb, p, eob, rows, n_next):
    beams = [B.Beam([], pp, e) for pp, e in zip(p, eob)]
    try:
        out = B.step(nb, beams, [B.Beam([], 0, False) for _ in range(n_next)], [np.asarray(r, np.float32) for r in rows])
    except B.Underflow:
        return -1, []
    return len(out), [(b.parent, b.token, B.p_bits(b.p), int(b.eob)) for b in out]


def constructed_steps():
    """(n_beams, p, eob, rows, n_next): ties inside the top-k scan, equal p across children and beams, eob beams tied with live
    ones, -inf and +inf logits, and random rows of ties at every beam count."""
    rng = np.random.default_rng(7)
    out = []
    tie = np.zeros((4, 40), np.float32)
    tie[:, [3, 17, 30, 31]] = 1.0                                   # four equal maxima per row, all beams alike
    out.append((4, [0.25] * 4, [0, 0, 0, 0], tie, 4))
    out.append((4, [0.25] * 4, [1, 0, 1, 0], tie, 4))               # eob beams at the live beams' p
    out.append((3, [0.5, 0.5], [0, 1], np.vstack([tie[0], tie[0]]), 1))
    inf = np.full((2, 64), -np.inf, np.float32)
    inf[:, :5] = [0.0, -1.0, 0.0, -2.0, -1.0]
    out.append((2, [0.5, 0.5], [0, 0], inf, 2))                     # -inf everywhere but five ids
    pinf = rng.standard_normal((2, 50)).astype(np.float32)
    pinf[0, 9] = np.inf
    out.append((2, [0.75, 0.25], [0, 0], pinf, 2))                  # +inf: the reference's max - max is NaN
    big = np.float32([3.0e38, -3.0e38, 1e-38, -1e-45, 0.0, -0.0] * 5).reshape(1, 30)
    out.append((5, [1.0], [0], big, 0))                             # finite extremes, a first step
    for t in range(60):
        nb = int(rng.integers(1, 9))
        nv = int(rng.integers(nb, 80))
        n_in = int(rng.integers(1, nb + 1))
        rows = rng.integers(-3, 3, size=(n_in, nv)).astype(np.float32) * np.float32(0.5)
        p = (rng.integers(1, 4, n_in) / 4).astype(np.float32).tolist()
        eob = [int(x) for x in rng.integers(0, 2, n_in)] if t % 2 else [0] * n_in
        if all(eob):
            eob[0] = 0
        out.append((nb, p, eob, rows, (0, 1, nb)[t % 3]))
    return out


def test_beam_step_matches_restatement(lib):
    for i, (nb, p, eob, rows, n_next) in enumerate(constructed_steps()):
        assert beam_step_c(lib, nb, p, eob, rows, n_next) == beam_step_py(nb, p, eob, rows, n_next), i


def test_beam_step_underflow_is_an_error(lib):
    """A beam whose second continuation's p underflows to 0 while the heap's front is still 0: the reference reads past its
    candidates; here the step returns -1."""
    row = np.full((2, 16), -200.0, np.float32)
    row[:, 0] = 0.0
    assert beam_step_py(2, [1e-30, 1e-30], [0, 0], row, 2)[0] == -1
    assert beam_step_c(lib, 2, [1e-30, 1e-30], [0, 0], row, 2)[0] == -1
    assert beam_step_c(lib, 2, [0.5, 0.5], [0, 0], np.zeros((2, 16), np.float32), 2)[0] == 2   # (and the same call works)


# ------------------------------------------------------------------------------------------ 3. re-parenting
def save(m, slot, tokens):
    st = m.save(slot)
    assert st.tokens == list(tokens)
    return bytes(st.data)


def test_reparent_copies_the_suffix(lib, model_dir):
    """Slot 0 evaluates X (300 tokens), slot 1 X[:280] and 30 other tokens.  Re-parenting 0 -> 1 over [280, 300) leaves slot 1's
    state (K / V of positions < 300, last logits and embeddings) byte-equal to slot 0's and to slot 2's, a fresh slot that
    evaluated X; the launch moves the rows of 20 positions (V: one 256-block), not the context's 512."""
    from ctransformers_b200 import Config, MultiLLM
    path, _ = modelcases.build("llama_tiny_q4km", model_dir)
    m = MultiLLM(str(path), n_slots=3, config=Config(context_length=512))
    x = modelcases.seeded_prompt("llama_tiny_q4km", 300, seed=5)
    y = x[:280] + modelcases.seeded_prompt("llama_tiny_q4km", 31, seed=6)[1:]
    m.eval({0: x, 1: y, 2: x}, batch_size=64)
    moved = lib.ctb_multi_reparent(m._m, 1, (C.c_int * 1)(0), (C.c_int * 1)(1), (C.c_int * 1)(280), (C.c_int * 1)(300))
    m._context[1] = list(x)
    want = save(m, 2, x)
    assert save(m, 0, x) == want
    assert save(m, 1, x) == want
    same(multi_state(m, 1)[0], multi_state(m, 2)[0], "re-parented slot's last logits")
    assert m.greedy([1]) == m.greedy([2])
    n_layer, n_kv, hd = 3, 4, 64
    assert moved == n_layer * n_kv * (20 * hd + hd * 256) * 2
    assert moved * 3 < n_layer * n_kv * (512 * hd + 512 * hd) * 2
    # a slot that is both a source and a destination is refused, and nothing moves
    assert lib.ctb_multi_reparent(m._m, 2, (C.c_int * 2)(0, 1), (C.c_int * 2)(1, 2), (C.c_int * 2)(0, 0), (C.c_int * 2)(300, 300)) == -1
    assert save(m, 2, x) == want


# ------------------------------------------------------------------------------------------ 4. refusals and the handle afterwards
def test_refusals_leave_the_handle_usable(lib, model_dir):
    name = "llama_tiny_q4km"
    m = handle(name, model_dir, 8)
    prompt = modelcases.prompt_for(name)
    with pytest.raises(ValueError):
        m.beam_search(prompt, 9, 4)
    with pytest.raises(ValueError):
        m.beam_search(prompt, 0, 4)
    with pytest.raises(ValueError):
        m.beam_search([], 2, 4)
    with pytest.raises(ValueError):
        m.beam_search(prompt, 2, m.context_length - len(prompt) + 1)
    off = (C.c_int * 2)(0, len(prompt))
    toks = (C.c_int * len(prompt))(*prompt)
    out_off, out_tok, out_p = (C.c_int * 2)(), (C.c_int * 64)(), (C.c_float * 1)()
    for nb, n_predict, o in ((9, 4, off), (0, 4, off), (2, m.context_length, off), (2, 4, (C.c_int * 2)(0, 0))):
        assert lib.ctb_multi_beam_search(m._m, 1, o, toks, nb, n_predict, 8, out_off, out_tok, out_p) == -1
    # the handle still gives the reference's greedy run (model_<name>.npz) in a slot a search used, and a search after it
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    m.reset(0)
    m.eval({0: gold["prompt"].tolist()}, batch_size=8)
    toks = []
    for _ in range(8):
        toks.append(m.greedy([0])[0])
        m.eval({0: [toks[-1]]})
    assert toks == gold["tokens"][:8].tolist()
    m.reset(0)
    response, p = m.beam_search(B.cases()[f"{name}_b2"][1], 2, B.N_PREDICT, batch_size=B.BATCH_SIZE)
    check(f"{name}_b2", response, p)
    assert all(not m.context(s) for s in range(2))
