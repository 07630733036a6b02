"""Multi-sequence decoding on the GPU (ctransformers_b200.MultiLLM, include/ctransformers_b200.h ctb_multi_*): after every eval,
each slot's logits, embeddings, greedy pick and sampler draw are bit-identical to a single-sequence LLM fed that slot's calls,
whatever the other slots do in the same launches — and therefore to the reference."""
import ctypes as C

import numpy as np
import pytest

import head_dims_refs as H
import modelcases
import q3k_refs as Q
import refs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("multi_seq_models")


def build(name, directory):
    if name in modelcases.CASES:
        return modelcases.build(name, directory)
    if name in H.all_cases():
        return H.build_model(name, directory)
    return Q.build_model(name, directory)


def arch_vocab(name):
    for table in (modelcases.CASES, H.all_cases(), Q.all_cases()):
        if name in table:
            return table[name][0], table[name][1].n_vocab
    raise KeyError(name)


def same(got, want, what):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ (first at {int(np.argmax(bad))}, max |d| {np.abs(got - want).max():.3e})"


def multi_state(m, slot):
    lg, em = m._lib.ctb_multi_logits(m._m, slot), m._lib.ctb_multi_embeddings(m._m, slot)
    assert lg and em, f"slot {slot} has no results"
    return np.ctypeslib.as_array(lg, (m.vocab_size,)).copy(), np.ctypeslib.as_array(em, (m.n_embd,)).copy()


def llm_state(llm):
    return (np.ctypeslib.as_array(llm.ctransformers_llm_logits_data(), (llm.vocab_size,)).copy(),
            np.array(llm.embeddings, np.float32))


def load(path, ctx):
    from ctransformers_b200 import AutoModelForCausalLM
    return AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)


def multi(path, ctx, n_slots):
    from ctransformers_b200 import Config, MultiLLM
    return MultiLLM(str(path), n_slots=n_slots, config=Config(context_length=ctx))


# ------------------------------------------------------------------------------------------ 1. the reference's digests
@pytest.mark.parametrize("name", ["llama_tiny_q4km", "llama_gqa_q5km", "falcon_tiny_q5km"])
def test_slots_against_reference_digests(name, model_dir):
    """Three slots run the model case's prompt at batch_size 8, 64 and 5 and N_NEW greedy steps, joining one after another among
    filler slots that decode random tokens; each equals the reference's run of that chunking."""
    path, ctx = build(name, model_dir)
    arch, n_vocab = arch_vocab(name)
    prompt = modelcases.prompt_for(name)
    m = multi(path, ctx, 6)
    rng = np.random.default_rng(3)
    targets = {1: 8, 3: 64, 4: 5}
    start_round = {1: 0, 3: 2, 4: 5}
    fillers = {0: 0, 2: 1, 5: 4}                          # filler slot -> round it starts
    runs = {s: {"toks": []} for s in targets}
    for rnd in range(max(start_round.values()) + modelcases.N_NEW + 1):
        by_bs = {}                                          # one eval call per batch size that starts a prompt this round
        decode = {}
        for s, bs in targets.items():
            if rnd == start_round[s]:
                by_bs.setdefault(bs, {})[s] = prompt
            elif start_round[s] < rnd <= start_round[s] + modelcases.N_NEW:
                t = m.greedy([s])[0]
                runs[s]["toks"].append(t)
                decode[s] = [t]
        for s, r0 in fillers.items():
            if rnd == r0:
                decode[s] = rng.integers(0, n_vocab, 9 + s).tolist()
            elif rnd > r0 and len(m.context(s)) < ctx - 1:
                decode[s] = [int(rng.integers(0, n_vocab))]
        calls = list(by_bs.items()) or [(8, {})]
        calls[0][1].update(decode)
        for bs, d in calls:
            m.eval(d, batch_size=bs)
            for s in d:
                if s in targets and rnd == start_round[s]:
                    runs[s]["first_logits"], runs[s]["first_embd"] = multi_state(m, s)
                if s in targets and rnd == start_round[s] + modelcases.N_NEW:
                    runs[s]["last_logits"] = multi_state(m, s)[0]
    gold = refs.golden_runs()
    for s, bs in targets.items():
        key = f"live_{name}_bs{bs}"
        assert runs[s]["toks"] == gold[f"{key}_tokens"].tolist(), f"slot {s} bs {bs}"
        for k in ("first_logits", "first_embd", "last_logits"):
            assert refs.digest(runs[s][k]) == str(gold[f"{key}_{k}"]), f"slot {s} bs {bs}: {k} is not the reference's"
    model = np.load(refs.GOLD / f"model_{name}.npz")
    r = runs[1]
    same(r["first_logits"], model["first_logits"], "first logits")
    same(r["first_embd"], model["first_embd"], "first embeddings")
    assert r["toks"] == model["tokens"][: modelcases.N_NEW].tolist()


# ------------------------------------------------------------------------------------------ 2. against single-sequence LLMs
class Mirror:
    """A MultiLLM and, per slot, a single-sequence LLM fed the same calls; every eval compares the evaluated slots."""

    def __init__(self, path, ctx, n_slots):
        self.path, self.ctx = path, ctx
        self.m = multi(path, ctx, n_slots)
        self.llms = {}

    def reset(self, s):
        self.m.reset(s)
        self.llms.pop(s, None)

    def eval(self, d, bs):
        self.m.eval(d, batch_size=bs)
        for s, toks in d.items():
            if s not in self.llms:
                self.llms[s] = load(self.path, self.ctx)
            self.llms[s].eval(toks, batch_size=bs)
        for s in d:
            lg, em = multi_state(self.m, s)
            want_lg, want_em = llm_state(self.llms[s])
            same(lg, want_lg, f"slot {s} logits after {len(self.m.context(s))} tokens")
            same(em, want_em, f"slot {s} embeddings")
        picks = self.m.greedy(list(d))
        for s, p in zip(d, picks):
            assert p == self.llms[s].sample(top_k=1, repetition_penalty=1.0, seed=0), f"slot {s} greedy pick"
        return dict(zip(d, picks))


@pytest.mark.parametrize("name", ["llama_wide_q4km", "llama_hd80_q4km_gqa", "llama_gqa_q3km", "falcon_tiny_q5km"])
def test_slots_against_single_sequence_llm(name, model_dir):
    """32 slots: prompts of 1, 2, 7, 31, 32, 33 and 70 tokens and random ones, at different batch sizes, joining while others
    decode; evals split across launches; slots finish, are reset and reused."""
    path, ctx = build(name, model_dir)
    _, n_vocab = arch_vocab(name)
    rng = np.random.default_rng(7)
    S = 32
    lengths = [1, 2, 7, 31, 32, 33, 70] + rng.integers(1, 40, S - 7).tolist()
    prompts = [rng.integers(0, n_vocab, n).tolist() for n in lengths]
    sizes = [8, 64, 5, 512, 3, 1]
    mir = Mirror(path, ctx, S)
    picks = {}
    # round 0: half the slots start, in two calls of different batch sizes
    picks.update(mir.eval({s: prompts[s] for s in range(0, 16, 2)}, 64))
    picks.update(mir.eval({s: prompts[s] for s in range(1, 16, 2)}, 5))
    for rnd in range(1, 7):
        d = {s: [picks[s]] for s in picks if len(mir.m.context(s)) < ctx - 8}
        if rnd == 2:                                        # the other half joins while the first decodes
            d.update({s: prompts[s] for s in range(16, S)})
        if rnd == 3:                                        # a multi-token continuation of one slot among single tokens
            d[5] = rng.integers(0, n_vocab, 6).tolist()
        if rnd == 4:                                        # slots finish, are reset and reused with new prompts
            for s in (0, 3, 6):
                mir.reset(s)
                picks.pop(s, None)
                d[s] = rng.integers(0, n_vocab, 20 + s).tolist()
        picks = {**picks, **mir.eval(d, sizes[rnd % len(sizes)])}
    assert mir.m.launches() > 0


# ------------------------------------------------------------------------------------------ 3. against the oracle
def test_slots_against_oracle(model_dir):
    """Three slots against one whole-model oracle each, value by value: a failure shows where it goes wrong."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    prompts = [modelcases.prompt_for(name), modelcases.long_prompt(name), modelcases.seeded_prompt(name, 12)]
    m = multi(path, ctx, 3)
    oracles = [refs.OracleModel(path, ctx) for _ in prompts]
    m.eval(dict(enumerate(prompts)), batch_size=8)
    for o, p in zip(oracles, prompts):
        o.eval(p, batch_size=8)
    for step in range(6):
        for s, o in enumerate(oracles):
            lg, em = multi_state(m, s)
            same(lg, o.logits, f"slot {s} step {step} logits")
            same(em, o.embd, f"slot {s} step {step} embeddings")
        picks = m.greedy([0, 1, 2])
        assert picks == [int(np.argmax(o.logits)) for o in oracles]
        m.eval({s: [t] for s, t in enumerate(picks)})
        for o, t in zip(oracles, picks):
            o.eval([t])


# ------------------------------------------------------------------------------------------ 4. one launch per lockstep step
@pytest.mark.parametrize("S", [5, 32])
def test_lockstep_decode_is_one_launch_per_step(S, model_dir):
    path, ctx = build("llama_tiny_q4km", model_dir)
    m = multi(path, ctx, S)
    rng = np.random.default_rng(S)
    m.eval({s: rng.integers(0, 1024, 3 + s).tolist() for s in range(S)}, batch_size=8)
    for _ in range(4):
        before = m.launches()
        picks = m.greedy(range(S))
        m.eval({s: [t] for s, t in enumerate(picks)})
        assert m.launches() == before + 1


# ------------------------------------------------------------------------------------------ 5. sampling
def test_sample_equals_single_sequence_draw(model_dir):
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    m = multi(path, ctx, 4)
    prompts = [modelcases.seeded_prompt(name, n, seed=n) for n in (5, 37, 12, 70)]
    llms = [load(path, ctx) for _ in prompts]
    m.eval(dict(enumerate(prompts)), batch_size=8)
    for llm, p in zip(llms, prompts):
        llm.eval(p, batch_size=8)
    for step in range(5):
        draws = {}
        for s, llm in enumerate(llms):
            kw = dict(top_k=40, top_p=0.9, temperature=0.8, seed=100 * step + s)
            draws[s] = m.sample(s, **kw)
            assert draws[s] == llm.sample(**kw), f"slot {s} step {step}"
        m.eval({s: [t] for s, t in draws.items()})
        for s, llm in enumerate(llms):
            llm.eval([draws[s]])



def test_one_slot_handle_equals_llm(model_dir):
    """A one-slot handle runs the multi-sequence path like any other: it evaluates, samples, saves and restores, and scores
    bit for bit as an LLM fed the same calls."""
    from ctransformers_b200.llm import _ints
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    m, llm = multi(path, ctx, 1), load(path, ctx)
    prompt = modelcases.seeded_prompt(name, 37, seed=37)
    m.eval({0: prompt}, batch_size=8)
    llm.eval(prompt, batch_size=8)
    for step in range(5):
        if step == 3:                                       # the slot starts over from its saved state
            saved = m.save(0)
            m.reset(0)
            m.restore(0, saved)
        lg, em = multi_state(m, 0)
        want_lg, want_em = llm_state(llm)
        same(lg, want_lg, f"logits at step {step}")
        same(em, want_em, f"embeddings at step {step}")
        kw = dict(top_k=40, top_p=0.9, temperature=0.8, seed=100 + step)
        t = m.sample(0, **kw)
        assert t == llm.sample(**kw), f"step {step}"
        m.eval({0: [t]})
        llm.eval([t])
    toks = modelcases.seeded_prompt(name, 11, seed=50)     # token i scored under the logits after token i - 1, as LLM.score scores
    lp, gr = np.zeros(len(toks)), np.zeros(len(toks), np.int32)
    assert m._lib.ctb_multi_eval_scored(m._m, 1, _ints([0]), _ints([0, len(toks)]), _ints(toks), _ints([len(m.context(0))]), 8,
                                        _ints(toks[1:] + [-1]), lp.ctypes.data_as(C.POINTER(C.c_double)), gr.ctypes.data_as(C.POINTER(C.c_int))) == 0
    want_lp, want_gr = llm.score(toks, batch_size=8)
    assert lp[:-1].tobytes() == want_lp[1:].tobytes()
    assert (gr[:-1] != 0).tolist() == want_gr[1:].tolist()

def test_generate_many_equals_generate(model_dir):
    """Four prompts through two slots: each result is what LLM.generate gives that prompt, greedy."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    m = multi(path, ctx, 2)
    prompts = [modelcases.seeded_prompt(name, n, seed=n) for n in (3, 40, 9, 21)]
    got = m.generate_many(prompts, 10, top_k=1, repetition_penalty=1.0)
    for p, g in zip(prompts, got):
        llm = load(path, ctx)
        want = []
        for t in llm.generate(p, top_k=1, repetition_penalty=1.0):
            want.append(t)
            if len(want) == 10:
                break
        assert g == want


# ------------------------------------------------------------------------------------------ 6. refusals
def test_legacy_type_is_refused(model_dir, capfd):
    from ctransformers_b200.lib import ConfigStruct, load_library
    path, ctx = build("llama_tiny_q4_0", model_dir)
    assert load_library().ctb_multi_create(str(path).encode(), b"gguf", ConfigStruct(ctx, 0, True, False), 4) is None
    assert "is not supported by the CUDA path" in capfd.readouterr().err


def test_long_context_is_refused(model_dir, capfd):
    from ctransformers_b200.lib import ConfigStruct, load_library
    path, _ = build("falcon_tiny_q5km", model_dir)
    assert load_library().ctb_multi_create(str(path).encode(), b"gguf", ConfigStruct(4096, 0, True, False), 2) is None
    err = capfd.readouterr().err
    assert "is not supported by the CUDA path" in err and "4096" in err


def test_slot_out_of_range(model_dir, capfd):
    path, ctx = build("llama_tiny_q4km", model_dir)
    m = multi(path, ctx, 2)
    with pytest.raises(IndexError):
        m.eval({2: [1, 2, 3]})
    lib = m._lib
    assert not lib.ctb_multi_eval(m._m, 1, (C.c_int * 1)(5), (C.c_int * 2)(0, 1), (C.c_int * 1)(1), (C.c_int * 1)(0), 8)
    assert "out of range" in capfd.readouterr().err
    assert lib.ctb_multi_greedy(m._m, 1, (C.c_int * 1)(-1), (C.c_int * 1)()) == -1
    assert lib.ctb_multi_reset(m._m, 2) == -1
    assert not lib.ctb_multi_logits(m._m, 7)


def test_llm_and_multi_llm_in_one_process(model_dir):
    """An LLM and a MultiLLM on the same file, their calls interleaved: both keep the reference's results."""
    name = "llama_tiny_q4km"
    path, ctx = build(name, model_dir)
    prompt = modelcases.prompt_for(name)
    llm = load(path, ctx)
    m = multi(path, ctx, 2)
    llm.eval(prompt, batch_size=8)
    m.eval({1: prompt}, batch_size=8)
    m.eval({0: modelcases.seeded_prompt(name, 30)}, batch_size=8)
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    same(llm_state(llm)[0], gold["first_logits"], "LLM first logits")
    same(multi_state(m, 1)[0], gold["first_logits"], "MultiLLM first logits")
    toks_a, toks_b = [], []
    for _ in range(modelcases.N_NEW):
        toks_a.append(llm.sample(top_k=1, repetition_penalty=1.0, seed=0))
        toks_b.append(m.greedy([1])[0])
        llm.eval([toks_a[-1]])
        m.eval({1: [toks_b[-1]], 0: [7]})
    assert toks_a == toks_b == gold["tokens"][: modelcases.N_NEW].tolist()
    same(llm_state(llm)[0], gold["last_logits"], "LLM last logits")
    same(multi_state(m, 1)[0], gold["last_logits"], "MultiLLM last logits")
