"""The last step of a token on the device, against plain numpy references (test_pick.py) at real vocabulary sizes and on ties,
signed zeros, infinities and NaN:

  * the greedy pick: k_argmax (look-ahead pick, un-fused PICK op, multi-sequence picks) and the step kernel's PH_PICK phase
    (ctb_llm_decode_greedy's token feedback) must both be the reference's top_k = 1 scan, with k_argmax's tie count;
  * the device top-k (k_sample_topk): the set of ids >= the k-th largest penalised logit, its count and its logits bit for bit;
  * the lazy sampler chain of ctransformers_llm_sample: the token ctb_sample (the host sampler, pinned to the reference) draws,
    answered on the device exactly where the cut is unambiguous;
  * whole models with vocabularies of 32000 and 65024: decode_greedy, lazy sampling and MultiLLM.greedy against an eager engine
    that picks with the scan on its host logits."""
import ctypes as C

import numpy as np
import pytest

from conftest import ptr
from test_pick import SIZES, F32, device_answers, penalise, ref_pick, ref_ties, ref_topk, sampler_vectors, vectors

pytestmark = pytest.mark.gpu
IP = C.POINTER(C.c_int)
FP = C.POINTER(C.c_float)
KS = [1, 2, 40, 127, 128]


def iptr(a):
    return a.ctypes.data_as(IP) if a is not None and len(a) else None


# ------------------------------------------------------------------------------------------------------------- greedy pick
def argmax_path(lib, path, x, state=(0, 0, 0, 0, 0)):
    x = np.ascontiguousarray(x, F32)
    out = np.zeros(6, np.int32)
    out[:5] = state
    assert lib.ctb_argmax_path(path, ptr(x), len(x), iptr(out)) == 0
    return out.tolist()


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("path", [0, 1], ids=["k_argmax", "k_step"])
def test_argmax_paths(lib, path, n):
    bad = []
    for i, (name, x) in enumerate(vectors(n)):
        pick = ref_pick(x)
        if path == 0:
            got, want = argmax_path(lib, 0, x)[:2], [pick, ref_ties(x, pick)]
        else:   # state {token, position, step, n_total, pick}: the pick becomes the token, out_tokens[step] and state[4]
            pos, step = 17 + i, i % 7
            got, want = argmax_path(lib, 1, x, (123, pos, step, 999, -7)), [pick, pos + 1, step + 1, pos + 2, pick, pick]
        if got != want:
            bad.append(f"{name}: {got} != {want}")
    assert not bad, bad


def test_argmax_path_refuses_what_it_cannot_take(lib):
    x = np.zeros(4, F32)
    out = np.zeros(6, np.int32)
    assert lib.ctb_argmax_path(0, ptr(x), 0, iptr(out)) == -1
    assert lib.ctb_argmax_path(1, ptr(x), 0, iptr(out)) == -1
    assert lib.ctb_argmax_path(2, ptr(x), 4, iptr(out)) == -1


# ------------------------------------------------------------------------------------------------------------- device top-k
def sample_topk(lib, x, last, penalty, k):
    x = np.ascontiguousarray(x, F32)
    last = np.ascontiguousarray(last, np.int32)
    ids, lg = np.full(256, -1, np.int32), np.zeros(256, F32)
    c = lib.ctb_sample_topk(ptr(x), len(x), iptr(last), len(last), penalty, k, iptr(ids), ptr(lg))
    return c, ids, lg


def topk_mismatch(lib, x, last, penalty, k):
    """What is wrong with the device's top-k of x (None: nothing)."""
    y = penalise(x, last, penalty)
    want = ref_topk(y, k)
    c, ids, lg = sample_topk(lib, x, last, penalty, k)
    if want is None:
        return None if c == -2 else f"returned {c}, not -2, with a NaN among the logits"
    if c != len(want):
        return f"count {c}, reference {len(want)}"
    got = ids[: min(c, 256)]
    if len(np.unique(got)) != len(got) or not np.isin(got, want).all() or (c <= 256 and len(got) != len(want)):
        return f"ids {sorted(got.tolist())[:8]}.. are not the reference set {want[:8].tolist()}.."
    if (lg[: len(got)].view(np.uint32) != y[got].view(np.uint32)).any():
        return "logits are not the penalised logits bit for bit"
    return None


@pytest.mark.parametrize("n", SIZES)
def test_sample_topk_vectors(lib, n):
    ks = KS + ([n + 1] if n + 1 <= 128 else [])
    bad = []
    for k in ks:
        for name, x in sampler_vectors(n, k):
            err = topk_mismatch(lib, x, [], 1.0, k)
            if err:
                bad.append(f"k {k}, {name}: {err}")
    assert not bad, bad


def windows(x, seed):
    """Repetition windows: none, one id, 64 with duplicates, 256 with negative ids and ids past the vocabulary, 257.  They hold the
    top logits, so that the penalty moves the cut."""
    n = len(x)
    rng = np.random.default_rng(seed)
    top = np.argsort(-x, kind="stable")[: min(n, 24)]
    w64 = np.concatenate([top[:16], top[:4], rng.integers(0, n, 44)])[:64]
    w256 = np.concatenate([top, [-1, -5, n, n + 7], top[:8], rng.integers(0, n, 256)])[:256]
    return {"none": [], "one": [int(top[0])], "w64": w64, "w256": w256, "w257": np.concatenate([w256, [0]])}


def penalty_vectors(n, penalty, seed):
    """A normal vector, one with exact zeros in the window, and one where the penalty makes a logit equal another one."""
    x = (np.random.default_rng(seed).standard_normal(n) * 0.5).astype(F32)
    z = x.copy()
    z[np.argsort(-x)[: min(n, 6)]] = 0.0
    z[: min(n, 3)] = -0.0
    eq = x.copy()
    if n >= 4:
        top = np.argsort(-x, kind="stable")
        eq[top[0]], eq[top[1]] = F32(4.0), F32(4.0) / F32(penalty)        # penalised top[0] (in every window) == top[1]
        eq[top[2]], eq[top[3]] = F32(-3.0), F32(-3.0) * F32(penalty)
    return [("normal", x), ("zeros", z), ("penalty_makes_equal", eq)]


@pytest.mark.parametrize("n", [2, 33, 1025, 32000, 65024])
def test_sample_topk_penalty(lib, n):
    bad, checked = [], 0
    for penalty in (1.0, 0.9, 1.1, 1.3):
        for vname, x in penalty_vectors(n, penalty, n):
            for wname, last in windows(x, n).items():
                for k in (1, 40, 128):
                    if len(last) > 256:
                        assert sample_topk(lib, x, last, penalty, k)[0] == -1
                        continue
                    err = topk_mismatch(lib, x, last, penalty, k)
                    checked += 1
                    if err:
                        bad.append(f"penalty {penalty}, {vname}, window {wname}, k {k}: {err}")
    assert not bad, bad
    assert checked > 100


def test_sample_topk_refuses_what_it_cannot_take(lib):
    x = np.arange(300, dtype=F32)
    for last, k in (([], 0), ([], 129), (list(range(257)), 40)):
        assert sample_topk(lib, x, last, 1.1, k)[0] == -1
    assert sample_topk(lib, x[:0], [], 1.0, 1)[0] == -1


# ------------------------------------------------------------------------------------------------------------- lazy sampler chain
# tests/golden/make_golden.py's settings (top_k, top_p, temperature, penalty, seed) and the common top-k 40 one without penalty
SETTINGS = [(40, 0.95, 0.8, 1.1, 1), (1, 1.0, 1.0, 1.0, 0), (5, 0.5, 1.3, 1.3, 7), (0, 0.9, 0.7, 1.0, 123), (1000, 1.0, 0.01, 1.2, 9),
            (40, 0.95, 0.8, 1.0, 3)]


def draw(lib, x, last, setting, seed):
    k, p, t, pen, _ = setting
    x = np.ascontiguousarray(x, F32)
    last = np.ascontiguousarray(last, np.int32)
    used = np.zeros(1, np.int32)
    dev = lib.ctb_sample_device(ptr(x), len(x), iptr(last), len(last), k, p, t, pen, seed, iptr(used))
    host = lib.ctb_sample(x.ctypes.data_as(FP), len(x), iptr(last), len(last), k, p, t, pen, seed)
    return dev, host, bool(used[0])


@pytest.mark.parametrize("n", [1, 2, 33, 1025, 32000, 65024, 151936])
def test_sample_device_is_the_host_sampler(lib, n):
    bad, on_device = [], 0
    for name, x in sampler_vectors(n, 40):
        for wname, last in (("none", []), ("w64", windows(np.nan_to_num(x), n)["w64"])):
            for s in SETTINGS:
                for seed in (s[4], s[4] + 1000):
                    dev, host, used = draw(lib, x, last, s, seed)
                    want_used = device_answers(x, last, s[0], s[3])
                    on_device += used
                    if dev != host or used != want_used:
                        bad.append(f"{name}, window {wname}, setting {s}, seed {seed}: device {dev} (on device {used}), host {host} "
                                   f"(on device expected {want_used})")
    assert not bad, bad[:20]
    assert on_device > 0


# ------------------------------------------------------------------------------------------------------------- whole models
CTX, N_STEPS = 64, 12
_models = {}


@pytest.fixture(scope="module")
def pick_model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("pick_models")


def model(name, d):
    """One-layer synthetic models with the vocabularies of Llama (32000) and Falcon (65024)."""
    from ctransformers_b200 import synth
    if name not in _models:
        path = d / f"{name}.gguf"
        if name == "llama_32000":
            synth.write_llama(path, synth.LlamaShape(n_vocab=32000, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=1, n_ctx_train=128),
                              "Q4_K_M", seed=21)
        else:
            synth.write_falcon(path, synth.FalconShape(n_vocab=65024, n_embd=256, n_head=4, n_head_kv=1, n_ff=1024, n_layer=1, n_ctx_train=128),
                               "Q5_K_M", seed=22)
        _models[name] = path
    return _models[name]


def load(path, eager):
    from ctransformers_b200 import AutoModelForCausalLM
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=CTX)
    if eager:
        _ = llm.logits   # host views from the start: every eval copies its logits, sample() runs on them like the reference's
    return llm


def host_logits(llm):
    return np.ctypeslib.as_array(llm.ctransformers_llm_logits_data(), (llm.vocab_size,)).astype(F32)


def prompt(path, seed):
    n_vocab = int(path.stem.split("_")[1])
    return np.random.default_rng(seed).integers(259, n_vocab, 8).tolist()


MODELS = ["llama_32000", "falcon_65024"]


@pytest.mark.parametrize("name", MODELS)
def test_decode_greedy_is_the_scan(name, pick_model_dir):
    path = model(name, pick_model_dir)
    toks = prompt(path, 1)
    a = load(path, eager=True)
    a.eval(toks)
    picks = [ref_pick(host_logits(a))]
    for _ in range(N_STEPS):
        a.eval([picks[-1]])
        picks.append(ref_pick(host_logits(a)))
    b = load(path, eager=False)
    b.eval(toks)
    out = (C.c_int * N_STEPS)()
    assert b.ctb_llm_decode_greedy(picks[0], len(toks), N_STEPS, out) > 0
    assert list(out) == picks[1:]


@pytest.mark.parametrize("name", MODELS)
def test_lazy_sampling_is_the_eager_engine(name, pick_model_dir):
    path = model(name, pick_model_dir)
    toks = prompt(path, 2)
    a, b = load(path, eager=False), load(path, eager=True)
    a.eval(toks)
    b.eval(toks)
    greedy = dict(top_k=1, repetition_penalty=1.0)
    sampled = dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1)
    plan = [greedy] * 4 + [sampled] * 4 + [greedy] * 3 + [dict(sampled, repetition_penalty=1.0)] * 3 + [greedy] * 2
    before = a.ctb_llm_device_samples()
    for i, kw in enumerate(plan):
        ta, tb = a.sample(seed=i, **kw), b.sample(seed=i, **kw)
        assert ta == tb, (i, kw)
        if kw is greedy:
            assert tb == ref_pick(host_logits(b))
        a.eval([ta])
        b.eval([tb])
    assert a.ctb_llm_device_samples() - before >= len(plan) - 2
    assert b.ctb_llm_device_samples() == 0


@pytest.mark.parametrize("name", MODELS)
def test_multi_greedy_is_the_llm(name, pick_model_dir):
    from ctransformers_b200 import Config, MultiLLM
    path = model(name, pick_model_dir)
    prompts = [prompt(path, 3), prompt(path, 4)[:5]]
    m = MultiLLM(str(path), n_slots=2, config=Config(context_length=CTX))
    single = [load(path, eager=True) for _ in prompts]
    m.eval({0: prompts[0], 1: prompts[1]})
    for llm, p in zip(single, prompts):
        llm.eval(p)
    for step in range(6):
        got = m.greedy([0, 1])
        assert got == [ref_pick(host_logits(llm)) for llm in single], step
        m.eval({0: [got[0]], 1: [got[1]]})
        for llm, t in zip(single, got):
            llm.eval([t])
