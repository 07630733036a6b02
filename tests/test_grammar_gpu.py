"""Grammar-constrained sampling on the GPU (k_grammar_mask, ctb_llm_sample_grammar, ctb_multi_sample_grammar_many): the device
mask equals the host mask (and the reference's) over whole vocabularies, LLM.generate(grammar=...) draws the reference's tokens,
MultiLLM draws per slot what LLM draws, and refusals leave the state and the handle usable."""
import itertools
import zlib
from pathlib import Path

import numpy as np
import pytest

import grammar_cases as G
from ctransformers_b200 import Config, Grammar, LLM, MultiLLM

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def runs():
    return np.load(GOLDEN / "grammar_runs.npz")


@pytest.fixture(scope="module")
def model_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("grammar_gpu_models")
    cache = {}

    def get(name):
        if name not in cache:
            path, ctx = G.build_model(name, d)
            cache[name] = (path, ctx, G.pieces_of(path))
        return cache[name]
    return get


def new_llm(model_files, name):
    path, ctx, _ = model_files(name)
    return LLM(str(path), config=Config(context_length=ctx))


def eos_of(name):
    return 2 if G.MODELS[name][0] == "llama" else 11


@pytest.mark.parametrize("model", sorted(G.MODELS))
def test_device_mask_equals_the_reference_along_every_golden_run(runs, model_files, model):
    llm = new_llm(model_files, model)
    pieces = model_files(model)[2]
    for gname, sname in itertools.product(G.RUN_GRAMMARS, G.SETTINGS):
        key = f"{model}__{gname}__{sname}"
        state = Grammar(G.GRAMMARS[gname]).start()
        for step, tok in enumerate(runs[f"{key}_tokens"]):
            want = np.unpackbits(runs[f"{key}_allowed"][step])[:llm.vocab_size].astype(bool)
            got = llm.grammar_mask(state)
            assert np.array_equal(got, want), (key, step, np.flatnonzero(got != want)[:10])
            assert np.array_equal(state.mask_pieces(pieces, eos_of(model)), want)
            if tok == eos_of(model) or (bool(runs[f"{key}_dead_end"]) and step == len(runs[f"{key}_tokens"]) - 1):
                break
            state.accept(llm, int(tok))
    assert llm.grammar_paths()["host_mask"] == 0


@pytest.mark.parametrize("model", ["llama_v32000", "falcon_v65024"])
@pytest.mark.parametrize("gname", ["json", "arithmetic", "list", "non_ascii", "operators"])
def test_device_mask_equals_host_along_random_walks(model_files, model, gname):
    llm = new_llm(model_files, model)
    pieces = model_files(model)[2]
    eos = eos_of(model)
    rng = np.random.default_rng(zlib.crc32(f"{model}/{gname}".encode()))
    partial_steps = 0
    for walk in range(3):
        state = Grammar(G.GRAMMARS[gname]).start()
        for step in range(24):
            host = state.mask_pieces(pieces, eos)
            assert np.array_equal(llm.grammar_mask(state), host), (walk, step)
            partial_steps += state.stacks[1][1] > 0
            ok = np.flatnonzero(host)
            ok = ok[ok != eos]
            if len(ok) == 0:
                break
            # prefer pieces that leave a partial UTF-8 sequence pending, so that those states are walked too
            part = [t for t in ok if pieces[t] and pieces[t][-1] >= 0x80]
            pool = part if part and rng.random() < 0.4 else ok
            # a piece with an overlong-encoded NUL passes the mask but no stack takes it (accept refuses, the state stays)
            for t in rng.permutation(pool):
                try:
                    state.accept(llm, int(t))
                    break
                except ValueError:
                    assert b"\x80" in pieces[t]
            else:
                break
    if gname in ("non_ascii", "list"):
        assert partial_steps > 0


@pytest.mark.parametrize("model", ["llama_v32000", "falcon_v65024"])
@pytest.mark.parametrize("lead", [b"\xc3", b"\xe6", b"\xe6\x97", b"\xf0", b"\xf0\x9f", b"\xf0\x9f\x98"])
def test_device_mask_with_each_partial_lead(model_files, model, lead):
    llm = new_llm(model_files, model)
    pieces = model_files(model)[2]
    for gname in ("non_ascii", "list", "json"):
        state = Grammar(G.GRAMMARS[gname]).start()
        if gname == "json":
            state.accept_piece(b'{"')
        try:
            state.accept_piece(lead)
        except ValueError:
            continue
        assert state.stacks[1][1] > 0
        assert np.array_equal(llm.grammar_mask(state), state.mask_pieces(pieces, eos_of(model))), gname


def test_bound_rows_are_answered_by_the_host(model_files):
    llm = new_llm(model_files, "llama_v32000")
    pieces = model_files("llama_v32000")[2]
    state = Grammar(G.DEEP).start()
    before = llm.grammar_paths()["host_mask"]
    got = llm.grammar_mask(state)
    assert llm.grammar_paths()["host_mask"] == before + 1
    host = state.mask_pieces(pieces, 2)
    assert np.array_equal(got, host)
    assert host[pieces.index(b"th")] and host[pieces.index(b"t")] and not host[pieces.index(b"the")]


@pytest.mark.parametrize("key", sorted(G.runs()))
def test_generate_draws_the_reference_tokens(runs, model_files, key):
    model, gname, sname = G.runs()[key]
    top_k, top_p, temp, pen, last_n, seed = G.SETTINGS[sname]
    llm = new_llm(model_files, model)
    want = runs[f"{key}_tokens"].tolist()
    gen = llm.generate(G.prompt(model), top_k=top_k, top_p=top_p, temperature=temp, repetition_penalty=pen, last_n_tokens=last_n,
                       seed=seed, grammar=G.GRAMMARS[gname])
    got = []
    if bool(runs[f"{key}_dead_end"]):
        # the last draw is a piece the mask allows but no stack takes (an overlong-encoded NUL): accepting it raises, where the
        # reference aborts
        with pytest.raises(ValueError):
            for t in gen:
                got.append(t)
        assert got == want[:-1]
    else:
        got = list(itertools.islice(gen, G.MAX_NEW))
        assert got == [t for t in want if t != eos_of(model)]
    # the steps with fewer allowed tokens than top_k took the host cut; the others the device
    allowed = [int(np.unpackbits(a)[:llm.vocab_size].sum()) for a in runs[f"{key}_allowed"]]
    few = sum(n < top_k for n in allowed)
    paths = llm.grammar_paths()
    assert paths["host_mask"] == 0
    assert paths["host_cut"] == few, (paths, allowed)
    assert paths["device"] == len(want) - few


def test_multi_sample_many_equals_llm_sample(model_files):
    name = "llama_tiny_q4km"
    path, ctx, pieces = model_files(name)
    n = 32
    m = MultiLLM(str(path), n_slots=n, config=Config(context_length=ctx))
    rng = np.random.default_rng(4)
    prompts = [[1] + rng.integers(259, 1000, 5 + i % 7).tolist() for i in range(n)]
    m.eval({s: prompts[s] for s in range(n)})
    kinds = [("json", "arithmetic", None)[s % 3] for s in range(n)]
    states = []
    for s, k in enumerate(kinds):
        if k is None:
            states.append(None)
            continue
        st = Grammar(G.GRAMMARS[k]).start()
        if s % 2:   # some states past their first characters
            st.accept_piece(b'{"' if k == "json" else b"x1")
        states.append(st)
    settings = dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1, seed=list(range(100, 100 + n)))
    before = m.grammar_paths()
    got = m.sample_many(list(range(n)), grammars=states, **settings)
    after = m.grammar_paths()
    assert sum(after[k] - before[k] for k in after) == sum(s is not None for s in states)
    for s in range(n):
        llm = LLM(str(path), config=Config(context_length=ctx))
        llm.eval(prompts[s])
        want = llm.sample(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1, seed=100 + s, grammar=states[s])
        assert got[s] == want, s
        if states[s] is not None:
            assert states[s].mask_pieces(pieces, 2)[got[s]]
    with pytest.raises(ValueError):
        m.sample_many([0, 1], grammars=[None])


def test_generate_many_equals_llm_generate(model_files):
    name = "llama_tiny_q4km"
    path, ctx, _ = model_files(name)
    m = MultiLLM(str(path), n_slots=8, config=Config(context_length=ctx))
    prompts = [G.prompt("llama_tiny_q4km"), [1, 300, 301, 302]]
    seeds = [1, 2, 3, 4]
    got = m.generate_many(prompts, 8, n=4, seeds=seeds, grammar=G.JSON)
    for i, p in enumerate(prompts):
        for j, seed in enumerate(seeds):
            llm = LLM(str(path), config=Config(context_length=ctx))
            want = list(itertools.islice(llm.generate(p, seed=seed, grammar=G.JSON), 8))
            assert got[i][j] == want, (i, j)


def test_grammar_sample_leaves_the_handle_as_without_it(model_files):
    name = "llama_tiny_q4km"
    a, b = new_llm(model_files, name), new_llm(model_files, name)
    p = G.prompt(name)
    for llm in (a, b):
        llm.eval(p)
    a.sample(seed=3, grammar=Grammar(G.JSON).start())
    assert a.sample(seed=5) == b.sample(seed=5)
    assert a.sample(top_k=1) == b.sample(top_k=1)
    for llm in (a, b):
        llm.eval([300])
    assert a.sample(top_k=1) == b.sample(top_k=1)
    assert list(a.logits) == list(b.logits)
    assert list(a.embeddings) == list(b.embeddings)
    # with a host view held, the mask runs on the host over that view
    s = Grammar(G.ARITHMETIC).start()
    assert a.sample(seed=9, grammar=s) == b.sample(seed=9, grammar=s)
    assert a.grammar_paths()["host_cut"] >= 1


def test_refusals_leave_the_state_and_handle_usable(model_files):
    name = "llama_tiny_q4km"
    llm = new_llm(model_files, name)
    pieces = model_files(name)[2]
    llm.eval(G.prompt(name))
    s = Grammar(G.FIXED).start()
    stacks = s.stacks
    with pytest.raises(ValueError):
        s.accept(llm, pieces.index(b"k"))      # "ok" must start with o
    with pytest.raises(ValueError):
        s.accept(llm, 2)                       # EOS before "ok"
    assert s.stacks == stacks
    nothing = Grammar(G.NOTHING).start()
    with pytest.raises(ValueError):
        llm.sample(grammar=nothing)
    assert not llm.grammar_mask(nothing).any()
    tok = llm.sample(seed=1, grammar=s)
    assert pieces[tok] in (b"o", b"ok")
    s.accept(llm, tok)
    assert llm.sample(top_k=1) >= 0
