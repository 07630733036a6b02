"""Sampling many rows at once on the device (k_sample_topk over a row dimension, ctb_multi_sample_many, MultiLLM.sample_many):
every row's device top-k is the single-row op's, every row's draw is the host sampler's (ctb_sample, pinned to the reference),
and every slot's draw is what a single-sequence LLM fed that slot's tokens returns, with the same arguments and seed."""
import ctypes as C
import itertools

import numpy as np
import pytest

import modelcases
from conftest import ptr
from test_pick import SIZES, F32, device_answers, penalise, ref_topk, sampler_vectors
from test_pick_gpu import SETTINGS, iptr, sample_topk, windows

pytestmark = pytest.mark.gpu
IP = C.POINTER(C.c_int)
FP = C.POINTER(C.c_float)
PENALTIES = (1.0, 0.9, 1.1, 1.3)
COMBOS = list(itertools.product(["none", "one", "w64", "w256", "w257"], PENALTIES, (1, 40, 128)))


def ints(v):
    return np.ascontiguousarray(v, np.int32)


def floats(v):
    return np.ascontiguousarray(v, F32)


def offsets(wins):
    return ints(np.concatenate([[0], np.cumsum([len(w) for w in wins])]))


def flat(wins):
    return ints(np.concatenate([np.asarray(w, np.int64) for w in wins] + [np.zeros(0, np.int64)]))


# ------------------------------------------------------------------------------------------------------------- rows op
def topk_rows(lib, xs, wins, pens, ks):
    x = floats(np.stack(xs))
    R, n = x.shape
    count, ids, lg = np.zeros(R, np.int32), np.full((R, 256), -1, np.int32), np.zeros((R, 256), F32)
    assert lib.ctb_sample_topk_rows(ptr(x), R, n, iptr(offsets(wins)), iptr(flat(wins)), floats(pens).ctypes.data_as(FP),
                                    iptr(ints(ks)), iptr(count), iptr(ids.reshape(-1)), lg.reshape(-1).ctypes.data_as(FP)) == 0
    return count, ids, lg


def rows_of(n):
    """(name, logits, window, penalty, k) rows with mixed settings: every vector of sampler_vectors under four of the (window,
    penalty, k) combinations, plus a k = 129 row."""
    out = []
    for v, (name, x) in enumerate(sampler_vectors(n, 40)):
        w = windows(np.nan_to_num(x), n + v)
        for j in range(4):
            wname, pen, k = COMBOS[(v * 7 + j * 13) % len(COMBOS)]
            out.append((f"{name}/{wname}/{pen}/{k}", x, w[wname], pen, k))
    x = sampler_vectors(n, 40)[0][1]
    out.append(("normal/k129", x, [], 1.0, 129))
    return out


@pytest.mark.parametrize("n", SIZES)
def test_topk_rows_are_the_single_row_op(lib, n):
    rows = rows_of(n)
    count, ids, lg = topk_rows(lib, [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows], [r[4] for r in rows])
    bad = []
    for i, (name, x, last, pen, k) in enumerate(rows):
        want_c, want_ids, want_lg = sample_topk(lib, x, last, pen, k)
        if count[i] != want_c:
            bad.append(f"{name}: count {count[i]}, alone {want_c}")
            continue
        if want_c <= 0:
            continue
        m = min(want_c, 256)
        got = ids[i, :m]
        if want_c <= 256:
            if sorted(got.tolist()) != sorted(want_ids[:m].tolist()):
                bad.append(f"{name}: ids are not the single-row op's")
            elif (lg[i, np.argsort(got)].view(np.uint32) != want_lg[:m][np.argsort(want_ids[:m])].view(np.uint32)).any():
                bad.append(f"{name}: logits are not the single-row op's bit for bit")
        elif len(np.unique(got)) != m or not np.isin(got, ref_topk(penalise(x, last, pen), k)).all():
            bad.append(f"{name}: the first 256 of {want_c} ids are not in the reference set")
    assert not bad, bad[:20]
    codes = set(count.tolist())
    assert -2 in codes and -1 in codes and max(codes) > 0      # a NaN row and refused rows next to answered ones, in one launch
    assert count[-1] == -1                                       # k = 129


def test_topk_rows_refuse_one_row_only(lib):
    x = np.random.default_rng(5).standard_normal((4, 1000)).astype(F32)
    x[2, 17] = np.nan
    wins = [[], list(range(257)), [3, 4], []]
    count, _, _ = topk_rows(lib, list(x), wins, [1.0, 1.1, 1.1, 1.0], [40, 40, 40, 129])
    assert count.tolist()[1:] == [-1, -2, -1]
    assert count[0] == sample_topk(lib, x[0], [], 1.0, 40)[0] == 40


# ------------------------------------------------------------------------------------------------------------- chain rows
@pytest.mark.parametrize("n", [1, 2, 33, 1025, 32000, 65024, 151936])
def test_sample_rows_are_the_host_sampler(lib, n):
    bad, on_device = [], 0
    for name, x in sampler_vectors(n, 40):
        rows = [(wname, last, s, seed) for wname, last in (("none", []), ("w64", windows(np.nan_to_num(x), n)["w64"]))
                for s in SETTINGS for seed in (s[4], s[4] + 1000)]
        R = len(rows)
        xs = floats(np.broadcast_to(x, (R, n)))
        wins = [r[1] for r in rows]
        col = lambda i: [r[2][i] for r in rows]
        tok, used = np.zeros(R, np.int32), np.zeros(R, np.int32)
        assert lib.ctb_sample_device_rows(ptr(xs), R, n, iptr(offsets(wins)), iptr(flat(wins)), iptr(ints(col(0))), floats(col(1)).ctypes.data_as(FP),
                                          floats(col(2)).ctypes.data_as(FP), floats(col(3)).ctypes.data_as(FP), iptr(ints([r[3] for r in rows])),
                                          iptr(tok), iptr(used)) == 0
        for i, (wname, last, s, seed) in enumerate(rows):
            k, p, t, pen, _ = s
            last = ints(last)
            host = lib.ctb_sample(floats(x).ctypes.data_as(FP), n, iptr(last), len(last), k, p, t, pen, seed)
            want_used = device_answers(x, last, k, pen)
            on_device += int(used[i])
            if tok[i] != host or bool(used[i]) != want_used:
                bad.append(f"{name}, window {wname}, setting {s}, seed {seed}: rows {tok[i]} (on device {used[i]}), host {host} "
                           f"(on device expected {want_used})")
    assert not bad, bad[:20]
    assert on_device > 0


# ------------------------------------------------------------------------------------------------------------- negative windows
def with_n_last(lib, fn, x, last, n_last, *rest):
    """fn(logits, n, last_tokens, n_last, *rest) with last_tokens holding `last` whatever n_last says."""
    x, last = floats(x), ints(last)
    return fn(ptr(x), len(x), iptr(last), n_last, *rest)


@pytest.mark.parametrize("n", [33, 32000])
def test_negative_window_is_no_window(lib, n):
    """n_last <= 0 is no window for the host sampler (sample_token); the device paths take it so too, with the pointer holding
    ids that a window would penalise."""
    x = np.random.default_rng(n).standard_normal(n).astype(F32)
    last = windows(x, n)["w256"]
    for k in (1, 2, 40, 128):
        got = [np.zeros(256, np.int32), np.zeros(256, F32)]
        want = [np.zeros(256, np.int32), np.zeros(256, F32)]
        c = with_n_last(lib, lib.ctb_sample_topk, x, last, -1, 1.3, k, iptr(got[0]), got[1].ctypes.data_as(FP))
        c0 = with_n_last(lib, lib.ctb_sample_topk, x, last, 0, 1.3, k, iptr(want[0]), want[1].ctypes.data_as(FP))
        assert c == c0 == min(k, n)
        assert sorted(got[0][:c].tolist()) == sorted(want[0][:c].tolist()), k
    used = np.zeros(1, np.int32)
    for s in SETTINGS:
        k, p, t, pen, seed = s
        dev = with_n_last(lib, lib.ctb_sample_device, x, last, -1, k, p, t, 1.3, seed, iptr(used))
        dev0 = with_n_last(lib, lib.ctb_sample_device, x, last, 0, k, p, t, 1.3, seed, iptr(used))
        host = lib.ctb_sample(floats(x).ctypes.data_as(FP), n, iptr(ints(last)), -1, k, p, t, 1.3, seed)
        assert dev == dev0 == host, s


def test_negative_window_through_llm_sample(model_dir):
    """ctransformers_llm_sample with n_last = -1 on logits still on the device, right after a draw with a full window: the same
    token as n_last = 0 and as the host sampler of an eager LLM."""
    from ctransformers_b200 import AutoModelForCausalLM
    path = model("llama_32000", model_dir)
    toks = np.random.default_rng(4).integers(259, 32000, 40).tolist()
    lazy = AutoModelForCausalLM.from_pretrained(str(path), context_length=CTX)
    eager = eager_llm(path, CTX)
    lazy.eval(toks)
    eager.eval(toks)
    x = np.ctypeslib.as_array(eager.ctransformers_llm_logits_data(), (32000,)).astype(F32)
    last = ints(windows(x, 3)["w256"])
    before = lazy.ctb_llm_device_samples()
    for seed in range(6):
        for k in (2, 40, 128):
            lazy.ctransformers_llm_sample(iptr(last), 256, k, 0.95, 0.8, 1.3, seed)      # leaves a 256-token window on the device
            got = lazy.ctransformers_llm_sample(iptr(last), -1, k, 0.95, 0.8, 1.3, seed)
            assert got == lazy.ctransformers_llm_sample(iptr(last), 0, k, 0.95, 0.8, 1.3, seed)
            assert got == eager.ctransformers_llm_sample(iptr(last), -1, k, 0.95, 0.8, 1.3, seed), (seed, k)
    assert lazy.ctb_llm_device_samples() > before


# ------------------------------------------------------------------------------------------------------------- whole models
CTX, N_STEPS = 320, 12
_models = {}


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("multi_sample_models")


def model(name, d):
    """One-layer synthetic models with the vocabularies of Llama (32000) and Falcon (65024), trained context 512."""
    from ctransformers_b200 import synth
    if name not in _models:
        path = d / f"{name}.gguf"
        if name == "llama_32000":
            synth.write_llama(path, synth.LlamaShape(n_vocab=32000, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=1, n_ctx_train=512),
                              "Q4_K_M", seed=31)
        else:
            synth.write_falcon(path, synth.FalconShape(n_vocab=65024, n_embd=256, n_head=4, n_head_kv=1, n_ff=1024, n_layer=1, n_ctx_train=512),
                               "Q5_K_M", seed=32)
        _models[name] = path
    return _models[name]


def eager_llm(path, ctx):
    from ctransformers_b200 import AutoModelForCausalLM
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    _ = llm.logits   # host views from the start: sample() runs the host sampler on them, as the reference does
    return llm


def multi(path, ctx, n_slots):
    from ctransformers_b200 import Config, MultiLLM
    return MultiLLM(str(path), n_slots=n_slots, config=Config(context_length=ctx))


# per slot: greedy; the config's defaults; penalty 1.3 over 64 tokens; top_k 0 (host path); top_p 0.5; a window of 300 (host path)
SLOT_SETTINGS = [dict(top_k=1, repetition_penalty=1.0), dict(), dict(repetition_penalty=1.3, last_n_tokens=64), dict(top_k=0),
                 dict(top_p=0.5), dict(last_n_tokens=300)]
KEYS = ("top_k", "top_p", "temperature", "repetition_penalty", "last_n_tokens")


@pytest.mark.parametrize("name", ["llama_32000", "falcon_65024"])
def test_sample_many_is_each_slots_llm(name, model_dir):
    path = model(name, model_dir)
    n_vocab = int(name.split("_")[1])
    rng = np.random.default_rng(9)
    prompts = [rng.integers(259, n_vocab, n).tolist() for n in (9, 40, 70, 17, 3, 280)]
    m = multi(path, CTX, len(prompts))
    llms = [eager_llm(path, CTX) for _ in prompts]
    m.eval(dict(enumerate(prompts)), batch_size=64)
    for llm, p in zip(llms, prompts):
        llm.eval(p, batch_size=64)
    cfg = m.config
    total = 0
    for step in range(N_STEPS):
        seeds = [1000 * step + s for s in range(len(prompts))]
        before = m.device_samples()
        got = m.sample_many(range(len(prompts)), seed=seeds, **{k: [st.get(k) for st in SLOT_SETTINGS] for k in KEYS})
        expect_dev = 0
        for s, (llm, st) in enumerate(zip(llms, SLOT_SETTINGS)):
            want = llm.sample(seed=seeds[s], **st)
            assert got[s] == want, f"step {step}, slot {s} {st}: {got[s]} != {want}"
            last_n = st.get("last_n_tokens", cfg.last_n_tokens)
            x = np.ctypeslib.as_array(llm.ctransformers_llm_logits_data(), (n_vocab,)).astype(F32)
            expect_dev += device_answers(x, m.context(s)[-last_n:], st.get("top_k", cfg.top_k), st.get("repetition_penalty", cfg.repetition_penalty))
        assert m.device_samples() - before >= expect_dev, step
        total += expect_dev
        m.eval({s: [t] for s, t in enumerate(got)})
        for llm, t in zip(llms, got):
            llm.eval([t])
    assert total > N_STEPS
    assert len(m.context(5)) > 256


def generate(path, ctx, prompt, n_new, seed):
    from ctransformers_b200 import AutoModelForCausalLM
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    out = []
    for t in llm.generate(prompt, seed=seed):
        out.append(t)
        if len(out) == n_new:
            break
    return out


@pytest.mark.parametrize("n", [1, 3])
def test_generate_many_sampled_equals_generate(n, model_dir):
    """Default sampling with seeds: each sample j of each prompt is LLM.generate of that prompt with seeds[j]."""
    name = "llama_tiny_q4km"
    path, ctx = modelcases.build(name, model_dir)
    m = multi(path, ctx, 4)
    prompts = [modelcases.seeded_prompt(name, k, seed=k) for k in (3, 40, 9, 21)]
    seeds = [11, 12, 11][:n]
    got = m.generate_many(prompts, 10, n=n, seeds=seeds)
    if n == 1:
        got = [[g] for g in got]
    for p, samples in zip(prompts, got):
        for j, g in enumerate(samples):
            assert g == generate(path, ctx, p, 10, seeds[j]), (p[:4], j)
        if n == 3:
            assert samples[0] == samples[2]


# ------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_draw_nothing(model_dir, capfd):
    name = "llama_tiny_q4km"
    path, ctx = modelcases.build(name, model_dir)
    prompts = [modelcases.seeded_prompt(name, k, seed=k) for k in (5, 30, 12)]

    def fresh():
        m = multi(path, ctx, 4)
        m.eval(dict(enumerate(prompts)), batch_size=8)
        return m

    kw = dict(top_k=[40, 1, 5], seed=[3, 4, 5])
    want = fresh().sample_many([0, 1, 2], **kw)
    m = fresh()
    lib = m._lib
    before = m.device_samples()
    with pytest.raises(IndexError):
        m.sample_many([0, 4, 1], **kw)
    with pytest.raises(RuntimeError):
        m.sample_many([0, 1, 0], **kw)
    with pytest.raises(RuntimeError):
        m.sample_many([0, 1, 3], **kw)            # slot 3 has evaluated nothing
    with pytest.raises(ValueError, match="top_k"):
        m.sample_many([0, 1, 2], top_k=[40, 1])
    with pytest.raises(ValueError, match="seed"):
        m.sample_many([0, 1], seed=[3, 4, 5])
    args = lambda *slots: (len(slots), (C.c_int * len(slots))(*slots), (C.c_int * (len(slots) + 1))(), None, (C.c_int * len(slots))(*[40] * len(slots)),
                           (C.c_float * len(slots))(*[0.95] * len(slots)), (C.c_float * len(slots))(*[0.8] * len(slots)),
                           (C.c_float * len(slots))(*[1.1] * len(slots)), (C.c_int * len(slots))(*range(len(slots))), (C.c_int * len(slots))())
    for slots in ((0, 7), (-1,), (2, 2), (1, 3)):
        assert lib.ctb_multi_sample_many(m._m, *args(*slots)) == -1, slots
    assert lib.ctb_multi_sample(m._m, 3, None, 0, 40, 0.95, 0.8, 1.1, 0) == -1
    err = capfd.readouterr().err
    assert "out of range" in err and "listed twice" in err and "no logits" in err
    assert m.device_samples() == before
    assert m.sample_many([0, 1, 2], **kw) == want
