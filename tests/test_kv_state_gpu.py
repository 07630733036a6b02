"""Sequence states on the GPU (MultiLLM.fork / save / restore, LLM.save_state / load_state, include/ctransformers_b200.h
ctb_multi_fork and ctb_*_state): a forked or restored sequence continues bit for bit as its uninterrupted run — against the
reference's digests, against single-sequence LLMs fed the whole history, and across handles of other context lengths."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import refs
from test_multi_seq_gpu import arch_vocab, build, llm_state, load, multi, multi_state, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("kv_state_models")


GREEDY = dict(top_k=1, repetition_penalty=1.0, seed=0)


# ------------------------------------------------------------------------------------------ 1. the reference's digests
@pytest.mark.parametrize("name", ["llama_tiny_q4km", "llama_gqa_q5km", "falcon_tiny_q5km"])
def test_fork_against_reference_digests(name, model_dir):
    """Slot 1 evaluates the prompt at batch_size 8 and is forked into slots 2, 3 and 4; the four then decode N_NEW greedy steps
    in shared evals while slots 0 and 5 decode random tokens.  Each equals the reference's run of that chunking."""
    path, ctx = build(name, model_dir)
    _, n_vocab = arch_vocab(name)
    gold = refs.golden_runs()
    key = f"live_{name}_bs8"
    m = multi(path, ctx, 6)
    rng = np.random.default_rng(4)
    m.eval({0: rng.integers(0, n_vocab, 11).tolist()}, batch_size=8)
    m.eval({1: modelcases.prompt_for(name), 5: rng.integers(0, n_vocab, 3).tolist()}, batch_size=8)
    team = [1, 2, 3, 4]
    m.fork(1, team[1:])
    for s in team:
        lg, em = multi_state(m, s)
        assert refs.digest(lg) == str(gold[f"{key}_first_logits"]), f"slot {s}: logits after the fork"
        assert refs.digest(em) == str(gold[f"{key}_first_embd"]), f"slot {s}: embeddings after the fork"
        assert m.context(s) == modelcases.prompt_for(name)
    toks = {s: [] for s in team}
    for _ in range(modelcases.N_NEW):
        picks = m.greedy(team)
        d = {s: [t] for s, t in zip(team, picks)}
        for s, t in zip(team, picks):
            toks[s].append(t)
        d.update({f: [int(rng.integers(0, n_vocab))] for f in (0, 5)})
        m.eval(d)
    for s in team:
        assert toks[s] == gold[f"{key}_tokens"].tolist(), f"slot {s}"
        assert refs.digest(multi_state(m, s)[0]) == str(gold[f"{key}_last_logits"]), f"slot {s}: last logits"


# ------------------------------------------------------------------------------------------ 2. against single-sequence LLMs
class ForkMirror:
    """A MultiLLM and, per slot, a single-sequence LLM fed that slot's whole call history; a forked slot's LLM replays the
    source's calls.  Every eval and fork compares the slots it touched."""

    def __init__(self, path, ctx, n_slots):
        self.path, self.ctx = path, ctx
        self.m = multi(path, ctx, n_slots)
        self.calls, self.llms = {}, {}

    def check(self, s):
        lg, em = multi_state(self.m, s)
        want_lg, want_em = llm_state(self.llms[s])
        same(lg, want_lg, f"slot {s} logits after {len(self.m.context(s))} tokens")
        same(em, want_em, f"slot {s} embeddings")
        assert self.m.context(s) == self.llms[s]._context

    def eval(self, d, bs):
        self.m.eval(d, batch_size=bs)
        for s, toks in d.items():
            if s not in self.llms:
                self.llms[s], self.calls[s] = load(self.path, self.ctx), []
            self.calls[s].append((list(toks), bs))
            self.llms[s].eval(toks, batch_size=bs)
        for s in d:
            self.check(s)

    def fork(self, src, dsts):
        self.m.fork(src, dsts)
        for d in dsts:
            self.calls[d] = list(self.calls[src])
            self.llms[d] = load(self.path, self.ctx)
            for toks, bs in self.calls[d]:
                self.llms[d].eval(toks, batch_size=bs)
            self.check(d)


@pytest.mark.parametrize("name", ["llama_gqa_q3km", "llama_hd80_q4km_gqa", "falcon_tiny_q5km"])
def test_forks_against_single_sequence_llm(name, model_dir):
    """Slots fork at random points, also over slots that hold longer histories, and diverge with seeded samples."""
    path, ctx = build(name, model_dir)
    _, n_vocab = arch_vocab(name)
    rng = np.random.default_rng(21)
    mir = ForkMirror(path, ctx, 8)
    mir.eval({0: rng.integers(0, n_vocab, 33).tolist(), 6: rng.integers(0, n_vocab, 50).tolist()}, 64)
    mir.eval({1: rng.integers(0, n_vocab, 7).tolist()}, 5)
    live = [0, 1, 6]
    for rnd in range(8):
        if rnd in (1, 3, 5):                                # fork a random live slot into one or two others, slot 6 included
            src = int(rng.choice(live))
            others = [s for s in range(8) if s != src and (s not in live or s == 6)]
            dsts = rng.choice(others, size=1 + rnd % 2, replace=False).tolist()
            mir.fork(src, dsts)
            live = sorted(set(live) | set(dsts))
        d = {}
        for s in live:
            if len(mir.m.context(s)) >= ctx - 8:
                continue
            kw = dict(top_k=40, top_p=0.9, temperature=0.8, seed=int(rng.integers(0, 1 << 30)))
            t = mir.m.sample(s, **kw)
            assert t == mir.llms[s].sample(**kw), f"slot {s} round {rnd}: sampled token"
            d[s] = [t] if rnd != 4 or s != live[0] else [t] + rng.integers(0, n_vocab, 5).tolist()
        mir.eval(d, [8, 64, 3][rnd % 3])


# ------------------------------------------------------------------------------------------ 3. round trips
def multi_steps(m, slot, n):
    toks = []
    for _ in range(n):
        toks.append(m.greedy([slot])[0])
        m.eval({slot: [toks[-1]]})
    return toks


def llm_steps(llm, n):
    toks = []
    for _ in range(n):
        toks.append(int(llm.sample(**GREEDY)))
        llm.eval([toks[-1]])
    return toks


def test_round_trips(model_dir):
    """A state saved after the prompt and 5 greedy steps continues, wherever it is restored, exactly as the reference's run:
    another slot, another MultiLLM of another context and slot count, an LLM, and from an LLM back into a MultiLLM."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    want = gold["tokens"].tolist()
    prompt = modelcases.prompt_for(name)
    k, rest = 5, modelcases.N_NEW - 5
    m = multi(path, ctx, 4)
    m.eval({0: prompt, 3: modelcases.long_prompt(name)[:50]}, batch_size=8)
    assert multi_steps(m, 0, k) == want[:k]
    st = m.save(0)
    assert st.n_past == len(prompt) + k and len(st.data) == m._lib.ctb_multi_state_size(m._m, st.n_past)
    # another slot of the same handle, over a longer history
    m.restore(3, st)
    assert m.context(3) == prompt + want[:k]
    assert multi_steps(m, 3, rest) == want[k:]
    same(multi_state(m, 3)[0], gold["last_logits"], "slot 3 last logits")
    # a second MultiLLM with another context length and slot count
    m2 = multi(path, ctx + 32, 3)
    m2.eval({2: modelcases.seeded_prompt(name, 80)}, batch_size=64)
    m2.restore(2, st)
    assert multi_steps(m2, 2, rest) == want[k:]
    same(multi_state(m2, 2)[0], gold["last_logits"], "second MultiLLM last logits")
    # MultiLLM -> LLM
    llm = load(path, ctx + 16)
    llm.load_state(st)
    same(llm_state(llm)[0], multi_state(m, 0)[0], "LLM logits right after the load")
    assert llm_steps(llm, rest) == want[k:]
    same(llm_state(llm)[0], gold["last_logits"], "LLM last logits")
    # LLM -> MultiLLM: a state saved by an LLM after 3 steps
    llm2 = load(path, ctx)
    llm2.eval(prompt, batch_size=8)
    assert llm_steps(llm2, 3) == want[:3]
    st2 = llm2.save_state()
    m.restore(1, st2)
    assert multi_steps(m, 1, modelcases.N_NEW - 3) == want[3:]
    same(multi_state(m, 1)[0], gold["last_logits"], "LLM -> MultiLLM last logits")
    # and the slot it was saved from went on untouched
    assert multi_steps(m, 0, rest) == want[k:]


def test_llm_state_moves_to_a_longer_context(model_dir):
    """An LLM at context 2304 with 2000 positions (batched prefill, ring attention) saves; an LLM at context 4096 (global-memory
    attention, no batched prefill) loads and continues exactly as the first one does."""
    name = "llama_tiny_q4km"
    path, _ = build(name, model_dir)
    a = load(path, 2304)
    a.eval(modelcases.seeded_prompt(name, 2000), batch_size=512)
    st = a.save_state()
    b = load(path, 4096)
    b.load_state(st)
    same(llm_state(b)[0], llm_state(a)[0], "logits right after the load")
    same(llm_state(b)[1], llm_state(a)[1], "embeddings right after the load")
    for step in range(8):
        ta, tb = llm_steps(a, 1), llm_steps(b, 1)
        assert ta == tb, f"step {step}"
        same(llm_state(b)[0], llm_state(a)[0], f"step {step} logits")


# ------------------------------------------------------------------------------------------ 4. restore over a dirty slot
@pytest.mark.parametrize("name", ["llama_tiny_q4km", "falcon_tiny_q5km"])
def test_restore_over_a_longer_history(name, model_dir):
    """The slot held 90 positions; after a restore of 37 its next eval is one 12-token chunk, whose attention rows run to
    n_total = 49 and read positions past each token with probability 0: they must be the zeros of a fresh slot."""
    path, ctx = build(name, model_dir)
    _, n_vocab = arch_vocab(name)
    prompt = modelcases.prompt_for(name)
    m = multi(path, ctx, 2)
    m.eval({0: prompt}, batch_size=8)
    st = m.save(0)
    rng = np.random.default_rng(2)
    m.eval({1: rng.integers(0, n_vocab, 90).tolist()}, batch_size=64)
    m.restore(1, st)
    chunk = rng.integers(0, n_vocab, 12).tolist()
    m.eval({1: chunk}, batch_size=64)
    fresh = load(path, ctx)
    fresh.eval(prompt, batch_size=8)
    fresh.eval(chunk, batch_size=64)
    lg, em = multi_state(m, 1)
    same(lg, llm_state(fresh)[0], "logits after the chunk")
    same(em, llm_state(fresh)[1], "embeddings after the chunk")
    # the same on an LLM that had the longer history
    llm = load(path, ctx)
    llm.eval(rng.integers(0, n_vocab, 90).tolist(), batch_size=64)
    llm.load_state(st)
    llm.eval(chunk, batch_size=64)
    same(llm_state(llm)[0], llm_state(fresh)[0], "LLM logits after the chunk")


# ------------------------------------------------------------------------------------------ 5. the LLM's greedy look-ahead
def test_llm_state_and_look_ahead(model_dir):
    """Save right after a greedy sample(), while the look-ahead step is in flight; load into an LLM whose own look-ahead is
    pending; both decode_greedy and eval + sample then continue with the uninterrupted run's tokens, and the look-ahead resumes."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    want = gold["tokens"].tolist()
    prompt = modelcases.prompt_for(name)
    a = load(path, ctx)
    a.eval(prompt, batch_size=8)
    assert llm_steps(a, 6) == want[:6]
    hits = a.ctb_llm_speculative_hits()
    assert hits > 0, "the look-ahead should be running by now"
    t = int(a.sample(**GREEDY))                            # the look-ahead for t at this position is in the stream
    assert t == want[6]
    st = a.save_state()
    assert st.tokens == prompt + want[:6]
    a.eval([t])
    assert a.ctb_llm_speculative_hits() == hits + 1
    assert llm_steps(a, 8) == want[7:15]

    b = load(path, ctx)
    b.eval(modelcases.long_prompt(name)[:40], batch_size=8)
    llm_steps(b, 5)
    b.sample(**GREEDY)                                     # b's own look-ahead is pending
    b.load_state(st)
    before = b.ctb_llm_speculative_hits()
    assert int(b.sample(**GREEDY)) == t
    b.eval([t])
    assert llm_steps(b, 8) == want[7:15]
    assert b.ctb_llm_speculative_hits() > before, "the look-ahead did not resume after the load"

    c = load(path, ctx)
    c.load_state(st)
    same(llm_state(c)[0], _logits_after(path, ctx, prompt + want[:6]), "logits right after the load")
    out = (C.c_int * 16)()
    assert c.ctb_llm_decode_greedy(t, st.n_past, 16, out) >= 0
    assert [t] + list(out[:16]) == want[6:23]
    same(llm_state(c)[0], _logits_after(path, ctx, prompt + want[:22]), "decode_greedy logits")


def _logits_after(path, ctx, tokens):
    """Logits of a fresh LLM after the prompt at batch_size 8 and then every further token as its own eval."""
    llm = load(path, ctx)
    n = modelcases.PROMPT_LEN
    llm.eval(tokens[:n], batch_size=8)
    for t in tokens[n:]:
        llm.eval([t])
    return llm_state(llm)[0]


# ------------------------------------------------------------------------------------------ 6. generate_many with forks
def test_generate_many_forks_each_prompt(model_dir):
    """n = 4 samples of one prompt on 4 slots: the prompt's 3 launches are paid once; each sample equals LLM.generate with its
    seed.  Then two prompts, n = 2, on 3 slots: the second waits for two free slots."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    kw = dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1)

    def generate(p, seed, n_new):
        llm, out = load(path, ctx), []
        for t in llm.generate(p, seed=seed, **kw):
            out.append(t)
            if len(out) == n_new:
                break
        return out

    m = multi(path, ctx, 4)
    prompt = modelcases.long_prompt(name)                  # 70 tokens: launches of 32 + 32 + 6
    seeds = [11, 12, 13, 14]
    evals, real_eval = [], m.eval

    def counting_eval(d, **a):
        before = m.launches()
        real_eval(d, **a)
        evals.append((sorted(d), m.launches() - before))
    m.eval = counting_eval
    got = m.generate_many([prompt], 10, n=4, seeds=seeds, **kw)
    assert evals[0] == ([0], 3), evals[0]
    assert all(n == 1 for _, n in evals[1:])
    assert got[0] == [generate(prompt, s, 10) for s in seeds]
    assert len({tuple(g) for g in got[0]}) > 1, "the seeds should draw different samples"

    m3 = multi(path, ctx, 3)
    prompts = [modelcases.seeded_prompt(name, 20, seed=5), modelcases.seeded_prompt(name, 9, seed=6)]
    got = m3.generate_many(prompts, 6, n=2, seeds=[3, 4], **kw)
    for p, g in zip(prompts, got):
        assert g == [generate(p, 3, 6), generate(p, 4, 6)]
    with pytest.raises(ValueError):
        m3.generate_many(prompts, 6, n=2, **kw)
    with pytest.raises(ValueError):
        m3.generate_many(prompts, 6, n=4, seeds=[1, 2, 3, 4], **kw)


# ------------------------------------------------------------------------------------------ 7. refusals
def test_refusals_leave_the_slot_as_it_was(model_dir, capfd):
    from ctransformers_b200 import SequenceState, synth
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    _, shape, ftype, _ = modelcases.CASES[name]
    twin = model_dir / "llama_tiny_q4km_twin.gguf"         # the same shape, other weights
    if not twin.exists():
        synth.write_llama(twin, shape, ftype, seed=12)
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    want = gold["tokens"].tolist()
    prompt = modelcases.prompt_for(name)

    m = multi(path, ctx, 2)
    m.eval({0: prompt}, batch_size=8)
    lib = m._lib
    capfd.readouterr()

    def refused(data, msg):
        data = bytes(data)
        assert lib.ctb_multi_restore(m._m, 0, data, len(data)) == -1
        assert msg in capfd.readouterr().err

    t = multi(twin, ctx, 2)
    t.eval({0: prompt}, batch_size=8)
    refused(t.save(0).data, "another model file")
    g = multi(build("llama_gqa_q5km", model_dir)[0], ctx, 2)
    g.eval({0: modelcases.prompt_for("llama_gqa_q5km")}, batch_size=8)
    refused(g.save(0).data, "another shape")
    long = multi(path, ctx + 64, 2)
    long.eval({0: modelcases.seeded_prompt(name, ctx + 10)}, batch_size=64)
    refused(long.save(0).data, "context length")
    good = bytearray(m.save(0).data)
    refused(good[:-4], "disagrees")
    bad = bytearray(good)
    bad[4] = 9
    refused(bad, "version 9")
    with pytest.raises(ValueError):
        m.restore(0, SequenceState([], bytes(good[:-4])))
    # an LLM refuses the same way
    llm = load(path, ctx)
    llm.eval(prompt, batch_size=8)
    assert llm.ctb_llm_load_state(bytes(bad), len(bad)) == -1 and "version 9" in capfd.readouterr().err
    long_st = long.save(0)
    with pytest.raises(RuntimeError):
        llm.load_state(long_st)
    assert "context length" in capfd.readouterr().err
    assert llm_steps(llm, modelcases.N_NEW) == want
    # the slot goes on as if nothing had been tried
    assert m.context(0) == prompt
    assert multi_steps(m, 0, modelcases.N_NEW) == want
    same(multi_state(m, 0)[0], gold["last_logits"], "last logits after the refusals")
    with pytest.raises(ValueError):
        m.fork(0, [0])
