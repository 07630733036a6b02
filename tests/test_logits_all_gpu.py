"""Every-token rows (the reference's logits_all) and their scores on the GPU: each row bit for bit the reference's (digests) and the
oracle's (orc_eval_rows) on every path an eval can take; nothing an ordinary eval leaves behind moves; MultiLLM rows equal a
single-sequence LLM's; the device scores equal float64 numpy over the same rows."""
import ctypes as C

import numpy as np
import pytest

import logits_all_cases as LA
import modelcases
import refs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("logits_all_gpu_models")


def same(got, want, what):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ (first at {int(np.argmax(bad))})"


def load(path, ctx):
    from ctransformers_b200 import AutoModelForCausalLM
    return AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)


def multi(path, ctx, n_slots):
    from ctransformers_b200 import Config, MultiLLM
    return MultiLLM(str(path), n_slots=n_slots, config=Config(context_length=ctx))


def paths(llm):
    out = (C.c_int * 8)()
    n = llm.ctb_llm_paths(out, 8)
    return dict(zip(["fused", "ring", "slots", "prefill", "prefill_launches", "single_steps"], list(out)[:n]))


def run_rows(llm, calls):
    """Each call as LLM.eval(..., logits_all=True); returns the rows of all calls and their chunk sizes."""
    rows, sizes = [], []
    for toks, bs in calls:
        llm.eval(toks, batch_size=bs, logits_all=True)
        rows.append(llm.all_logits.copy())
        sizes += LA.chunk_sizes(len(toks), bs, llm.context_length)
    return np.concatenate(rows), sizes


# ------------------------------------------------------------------------------------------ 1. every path, against the reference
PATHS = {
    "default": ({}, None),
    "no_prefill": ({"CTB_NO_PREFILL": "1"}, None),
    "unfused": ({"CTB_STEP_FUSE": "0"}, None),
    "ctx4096": ({}, 4096),
}
ORACLE_MAX = 200   # tokens up to which the rows are also compared with the oracle, value by value


def check_run(key, model_dir, monkeypatch, env, ctx_override):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    name, calls = LA.runs()[key]
    path, ctx = LA.build(name, model_dir)
    ctx = ctx_override or ctx
    llm = load(path, ctx)
    before = paths(llm)
    rows, sizes = run_rows(llm, calls)
    after = paths(llm)
    gold = LA.golden()
    if ctx_override is None:
        assert LA.digests(rows, sizes) == gold[f"{key}_chunks"].tolist(), f"{key}: rows are not the reference's"
    if sum(len(t) for t, _ in calls) <= ORACLE_MAX:
        model = refs.OracleModel(path, ctx)
        want = np.concatenate([b for toks, bs in calls for b in LA.oracle_rows(model, toks, bs, ctx)])
        same(rows, want, f"{key} rows against the oracle")
    return before, after


@pytest.mark.parametrize("key", list(LA.runs()))
def test_rows_match_reference(key, model_dir, monkeypatch):
    before, after = check_run(key, model_dir, monkeypatch, {}, None)
    name = LA.runs()[key][0]
    legacy = not (LA._table(name)[2].startswith("Q3_K") or LA._table(name)[2].endswith("_M"))
    if legacy:
        assert after["prefill"] == 0 and after["single_steps"] > before["single_steps"], "legacy layer matrices: single-token path"
    else:
        assert after["prefill_launches"] > before["prefill_launches"], "K-quant layers: batched path"


@pytest.mark.parametrize("variant", ["no_prefill", "unfused", "ctx4096"])
@pytest.mark.parametrize("key", [f"{n}_bs{bs}" for n in ("llama_tiny_q4km", "llama_gqa_q5km", "falcon_tiny_q5km", "llama_gqa_q3km")
                                 for bs in (8, 64, 5)] + [LA.OVERFLOW])
def test_rows_on_every_path(key, variant, model_dir, monkeypatch):
    env, ctx = PATHS[variant]
    before, after = check_run(key, model_dir, monkeypatch, env, ctx)
    if variant == "no_prefill" or variant == "ctx4096":
        assert after["prefill_launches"] == before["prefill_launches"] and after["single_steps"] > before["single_steps"]
    if variant == "unfused":
        assert after["fused"] == 0


# ------------------------------------------------------------------------------------------ 2. nothing else moves
def snapshot(llm):
    return np.array(llm.logits, np.float32), np.array(llm.embeddings, np.float32)


@pytest.mark.parametrize("name", ["llama_tiny_q4km", "falcon_tiny_q5km", "llama_tiny_q4_0"])
def test_rows_and_scores_change_nothing_else(name, model_dir):
    """Two LLMs fed the same calls, one with rows or scores on every other call: logits, embeddings, greedy picks (with the
    look-ahead in flight after a streak), seeded draws and the state round trip stay the same bits."""
    path, ctx = modelcases.build(name, model_dir)
    a, b = load(path, ctx), load(path, ctx)
    prompt = modelcases.prompt_for(name)
    a.eval(prompt, batch_size=8)
    b.eval(prompt, batch_size=8, logits_all=True)
    for x, y in zip(snapshot(a), snapshot(b)):
        same(x, y, "after the prompt")
    for step in range(8):   # greedy: from the third step on the look-ahead step is in flight when the next eval arrives
        ta = a.sample(top_k=1, repetition_penalty=1.0, seed=0)
        tb = b.sample(top_k=1, repetition_penalty=1.0, seed=0)
        assert ta == tb, f"greedy step {step}"
        a.eval([ta])
        if step % 3 == 0:
            b.eval([tb], logits_all=True)
            same(b.all_logits[0], snapshot(a)[0], f"step {step} row")
        elif step % 3 == 1:
            b.score([tb])
        else:
            b.eval([tb])
        for x, y in zip(snapshot(a), snapshot(b)):
            same(x, y, f"step {step}")
    assert a.sample(seed=7) == b.sample(seed=7)
    st_a, st_b = a.save_state(), b.save_state()
    a.load_state(st_a)
    b.load_state(st_b)
    more = modelcases.seeded_prompt(name, 9, seed=3)[1:]
    a.eval(more, batch_size=5)
    lp, gr = b.score(more, batch_size=5)
    for x, y in zip(snapshot(a), snapshot(b)):
        same(x, y, "after load_state")
    assert a.sample(top_k=1, repetition_penalty=1.0, seed=0) == b.sample(top_k=1, repetition_penalty=1.0, seed=0)


# ------------------------------------------------------------------------------------------ 3. multi-sequence
@pytest.mark.parametrize("name", ["llama_tiny_q4km", "llama_gqa_q5km", "llama_gqa_q3km", "falcon_tiny_q5km"])
def test_multi_rows_equal_single_sequence_rows(name, model_dir):
    path, ctx = LA.build(name, model_dir)
    n_vocab = LA.n_vocab(name)
    rng = np.random.default_rng(11)
    m = multi(path, ctx, 6)
    llms = {}
    prompts = {s: rng.integers(0, n_vocab, n).tolist() for s, n in enumerate((1, 7, 33, 40, 3, 70))}
    rounds = [({0: prompts[0], 2: prompts[2], 5: prompts[5]}, 8), ({1: prompts[1], 3: prompts[3], 4: prompts[4]}, 5)]
    for r in range(4):
        rounds.append(({s: rng.integers(0, n_vocab, 1 + (s + r) % 3).tolist() for s in range(6)}, 64))
    for d, bs in rounds:
        m.eval(d, batch_size=bs, logits_all=True)
        for s, toks in d.items():
            llm = llms.setdefault(s, load(path, ctx))
            llm.eval(toks, batch_size=bs, logits_all=True)
            same(m.all_logits[s], llm.all_logits, f"slot {s} rows after {len(m.context(s))} tokens")
    # a plain eval afterwards is untouched
    d = {s: [int(rng.integers(0, n_vocab))] for s in range(6)}
    m.eval(d)
    for s, toks in d.items():
        llms[s].eval(toks)
        same(np.ctypeslib.as_array(m._lib.ctb_multi_logits(m._m, s), (n_vocab,)), snapshot(llms[s])[0], f"slot {s} logits")


# ------------------------------------------------------------------------------------------ 4. scores against float64 numpy
def close(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    both_nan = np.isnan(got) & np.isnan(want)
    same_inf = np.isinf(want) & (got == want)
    ok = both_nan | same_inf | (np.abs(got - want) <= 1e-9)
    assert ok.all(), f"{what}: {int((~ok).sum())} differ, first at {int(np.argmax(~ok))}: {got[~ok][:3]} vs {want[~ok][:3]}"


def vocab_model(n_vocab, directory):
    from ctransformers_b200 import synth
    path = directory / f"llama_v{n_vocab}.gguf"
    if not path.exists():
        synth.write_llama(path, synth.LlamaShape(n_vocab=n_vocab, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256),
                          "Q4_K_M", seed=5)
    return path


@pytest.mark.parametrize("n_vocab", [1024, 32000, 65024])
def test_score_and_perplexity_against_numpy(n_vocab, model_dir):
    path = vocab_model(n_vocab, model_dir)
    ctx = 128
    rng = np.random.default_rng(n_vocab)
    toks = [1] + rng.integers(3, n_vocab, 70).tolist()
    a, b = load(path, ctx), load(path, ctx)
    a.eval(toks[:10], batch_size=8, logits_all=True)
    ctx_rows = a.all_logits
    a.eval(toks[10:], batch_size=8, logits_all=True)
    rows = np.concatenate([ctx_rows, a.all_logits])
    lp, gr = b.score(toks[:10], batch_size=8)
    assert np.isnan(lp[0]) and not gr[0]
    lp2, gr2 = b.score(toks[10:], batch_size=8)       # the first token from the kept last logits
    want_lp, want_gr = LA.logprob_ref(rows[:-1], toks[1:])
    close(np.concatenate([lp[1:], lp2]), want_lp, "logprob")
    assert (np.concatenate([gr[1:], gr2]) == (want_gr != 0)).all()
    c, d = load(path, ctx), load(path, ctx)
    ppl = c.perplexity(toks, batch_size=8)
    d.eval(toks, batch_size=8, logits_all=True)           # the same chunking as perplexity's one call
    ref_lp, _ = LA.logprob_ref(d.all_logits[:-1], toks[1:])
    assert abs(np.log(ppl) + np.mean(ref_lp)) <= 1e-9


@pytest.mark.parametrize("n_vocab", [32000, 65024])
def test_row_logprob_on_adversarial_rows(n_vocab):
    from ctransformers_b200.lib import load_library
    lib = load_library()
    rng = np.random.default_rng(n_vocab)
    rows = (rng.standard_normal((10, n_vocab)) * 4).astype(np.float32)
    rows[1, [5, 900, n_vocab - 1]] = rows[1].max() + 1          # ties at the maximum
    rows[2, 77] = np.nan
    rows[3, 0] = np.nan
    rows[4, [3, n_vocab - 2]] = np.inf
    rows[5, :] = -np.inf
    rows[6, ::2] = -np.inf
    rows[7, :] = 0.0
    rows[7, 11] = -0.0
    rows[8] = np.float32(3e38) * np.sign(rows[8])                # huge finite values
    targets = [0, 900, 77, 1, 3, 2, 1, 11, 5, -1]
    lp, gr = np.zeros(10), np.zeros(10, np.int32)
    assert lib.ctb_row_logprob(rows.ctypes.data_as(C.c_void_p), 10, n_vocab, (C.c_int * 10)(*targets), lp.ctypes.data_as(C.POINTER(C.c_double)),
                               gr.ctypes.data_as(C.POINTER(C.c_int))) == 0
    want_lp, want_gr = LA.logprob_ref(rows, targets)
    close(lp, want_lp, "logprob")
    assert gr.tolist() == want_gr.tolist()
    assert gr[1] == 0 and LA.greedy_ref(rows[1]) == 5


def test_score_many_against_single_sequence_rows(model_dir):
    name = "llama_tiny_q4km"
    path, ctx = modelcases.build(name, model_dir)
    rng = np.random.default_rng(4)
    reqs = [([1] + rng.integers(3, 1024, int(rng.integers(0, 40))).tolist(), rng.integers(3, 1024, int(rng.integers(1, 12))).tolist())
            for _ in range(32)]
    reqs[3] = (reqs[3][0], [])   # replaced below: a continuation of the greedy picks
    llm = load(path, ctx)
    llm.eval(reqs[3][0], logits_all=True)
    greedy = []
    for _ in range(5):
        greedy.append(llm.sample(top_k=1, repetition_penalty=1.0, seed=0))
        llm.eval([greedy[-1]])
    reqs[3] = (reqs[3][0], greedy)
    m = multi(path, ctx, 8)
    before = m.launches()
    got = m.score_many(reqs)
    assert m.launches() - before < sum(len(c) + len(k) for c, k in reqs) // 8
    for i, (c, k) in enumerate(reqs):
        one = load(path, ctx)
        whole = c + k
        one.eval(whole[:-1], batch_size=8, logits_all=True)
        lp, gr = LA.logprob_ref(one.all_logits[len(c) - 1:], k)
        assert abs(got[i][0] - float(np.sum(lp))) <= 1e-9 * max(1, len(k)), i
        assert got[i][1] == bool(np.all(gr != 0)), i
    assert got[3][1]


# ------------------------------------------------------------------------------------------ 5. refusals
def test_out_of_range_targets_are_refused(model_dir, capfd):
    name = "llama_tiny_q4km"
    path, ctx = modelcases.build(name, model_dir)
    llm, fresh = load(path, ctx), load(path, ctx)
    toks = modelcases.prompt_for(name)[:12]
    lp, gr = np.zeros(12), np.zeros(12, np.int32)
    for bad in (1024, -2):
        targets = list(toks[1:]) + [bad]
        rc = llm.ctb_llm_batch_eval_scored((C.c_int * 12)(*toks), 12, 0, 8, (C.c_int * 12)(*targets), lp.ctypes.data_as(C.POINTER(C.c_double)),
                                           gr.ctypes.data_as(C.POINTER(C.c_int)))
        assert rc == -1
        assert "out of range" in capfd.readouterr().err
    llm.eval(toks, logits_all=True)                     # the handle evaluated nothing and stays usable
    fresh.eval(toks, logits_all=True)
    same(llm.all_logits, fresh.all_logits, "rows after a refusal")
    m = multi(path, ctx, 2)
    rc = m._lib.ctb_multi_eval_scored(m._m, 1, (C.c_int * 1)(0), (C.c_int * 2)(0, 3), (C.c_int * 3)(1, 2, 3), (C.c_int * 1)(0), 8,
                                      (C.c_int * 3)(2, 3, 5000), lp.ctypes.data_as(C.POINTER(C.c_double)), gr.ctypes.data_as(C.POINTER(C.c_int)))
    assert rc == -1 and "out of range" in capfd.readouterr().err
    m.eval({0: toks}, logits_all=True)
    same(m.all_logits[0], fresh.all_logits, "multi rows after a refusal")
