"""CPU checks of the every-token rows (the reference's logits_all) and their scores: the oracle's rows against the digests of the
reference's, the float64 log-softmax reference on rows that are not all finite, and the argument checks of the Python surface."""
import ctypes as C

import numpy as np
import pytest

import logits_all_cases as LA
import modelcases
import refs


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("logits_all_models")


# ------------------------------------------------------------------------------------------ 1. the oracle's rows are the reference's
@pytest.mark.parametrize("key", list(LA.runs()))
def test_oracle_rows_match_reference_digests(key, model_dir):
    name, calls = LA.runs()[key]
    path, ctx = LA.build(name, model_dir)
    model = refs.OracleModel(path, ctx)
    got = []
    for toks, bs in calls:
        blocks = LA.oracle_rows(model, toks, bs, ctx)
        got += [refs.digest(b.reshape(-1)) for b in blocks]
        last = blocks[-1][-1]
    gold = LA.golden()
    assert got == gold[f"{key}_chunks"].tolist()
    assert np.array_equal(last.view(np.uint32), gold[f"{key}_last_row"].view(np.uint32))


@pytest.mark.parametrize("name", list(modelcases.CASES))
def test_last_row_is_the_golden_first_logits(name, model_dir):
    """The last row of the prompt eval at batch_size 8 is the logits the reference's ordinary eval leaves (model_<name>.npz)."""
    path, ctx = modelcases.build(name, model_dir)
    model = refs.OracleModel(path, ctx)
    gold = np.load(refs.GOLD / f"model_{name}.npz")
    blocks = LA.oracle_rows(model, gold["prompt"].tolist(), 8, ctx)
    assert np.array_equal(blocks[-1][-1].view(np.uint32), gold["first_logits"].view(np.uint32))
    assert np.array_equal(model.embd.view(np.uint32), gold["first_embd"].view(np.uint32))
    toks, cur = [], blocks[-1][-1]
    for _ in range(4):   # greedy steps through orc_eval_rows: the single row of each is the ordinary eval's
        toks.append(LA.greedy_ref(cur))
        cur = LA.oracle_rows(model, [toks[-1]], 8, ctx)[0][0]
    assert toks == gold["tokens"][:4].tolist()


# ------------------------------------------------------------------------------------------ 2. the float64 reference of the scores
def test_logprob_ref_on_finite_rows():
    rng = np.random.default_rng(1)
    rows = (rng.standard_normal((4, 1000)) * 5).astype(np.float32)
    t = [3, 999, -1, 0]
    lp, gr = LA.logprob_ref(rows, t)
    for r in (0, 1, 3):
        x = rows[r].astype(np.float64)
        want = x[t[r]] - np.log(np.sum(np.exp(x)))
        assert abs(lp[r] - want) < 1e-12
        assert gr[r] == int(np.argmax(rows[r]) == t[r])
    assert lp[2] == 0 and gr[2] == 0
    assert np.isclose(np.sum(np.exp([LA.logprob_ref(rows[:1], [i])[0][0] for i in range(1000)])), 1.0, atol=1e-12)


def test_logprob_ref_on_rows_that_are_not_finite():
    row = np.array([0.0, 1.0, 1.0, -np.inf, 0.5], np.float32)
    lp, gr = LA.logprob_ref([row] * 5, [0, 1, 2, 3, 4])
    assert lp[3] == -np.inf
    assert lp[1] == lp[2] and gr.tolist() == [0, 1, 0, 0, 0]           # a tie: the lowest id is the greedy pick
    inf = np.array([np.inf, 2.0, np.inf, -np.inf], np.float32)
    lp, gr = LA.logprob_ref([inf] * 2, [2, 1])
    assert lp[0] == -np.log(2.0) and lp[1] == -np.inf and gr.tolist() == [0, 0]
    nan = np.array([1.0, np.nan, 3.0], np.float32)
    lp, gr = LA.logprob_ref([nan, nan], [2, 1])
    assert np.isnan(lp).all() and gr.tolist() == [1, 0]               # NaN never wins the pick
    lp, gr = LA.logprob_ref([np.array([np.nan, 3.0], np.float32)], [0])
    assert np.isnan(lp[0]) and gr[0] == 1                               # NaN at id 0 keeps id 0
    lp, gr = LA.logprob_ref([np.full(4, -np.inf, np.float32)], [2])
    assert np.isnan(lp[0]) and gr[0] == 0                               # nothing above -inf: id 0
    lp, gr = LA.logprob_ref([np.array([-0.0, 0.0], np.float32)], [1])
    assert lp[0] == -np.log(2.0) and gr[0] == 0                         # signed zeros are equal


# ------------------------------------------------------------------------------------------ 3. argument checks without a GPU
class StubLib:
    """Answers the handful of calls the argument checks may make before the library would run anything."""

    def __init__(self):
        self.calls = []

    def ctransformers_llm_vocab_size(self, llm):
        return 100

    def ctransformers_llm_context_length(self, llm):
        return 64

    def __getattr__(self, name):
        def record(*args):
            self.calls.append(name)
            return -1
        return record


def stub_llm():
    from ctransformers_b200 import LLM
    from ctransformers_b200.llm import Config
    llm = LLM.__new__(LLM)
    llm.__dict__.update(_lib=StubLib(), _llm=1, _context=[], _config=Config())
    return llm


def stub_multi(n_slots=2):
    from ctransformers_b200 import MultiLLM
    from ctransformers_b200.llm import Config
    m = MultiLLM.__new__(MultiLLM)
    m.__dict__.update(_lib=StubLib(), _m=None, _config=Config(), n_slots=n_slots, vocab_size=100, context_length=64,
                      _context=[[] for _ in range(n_slots)])
    return m


@pytest.mark.parametrize("bad", [[1, 100], [-1], [5, 2, 1000]])
def test_llm_refuses_token_ids_out_of_range(bad):
    llm = stub_llm()
    for call in (lambda: llm.score(bad), lambda: llm.perplexity(bad), lambda: llm.eval(bad, logits_all=True)):
        with pytest.raises(ValueError, match="out of range"):
            call()
    assert llm._lib.calls == [] and llm._context == []


def test_score_many_refuses_bad_requests():
    m = stub_multi()
    for reqs, what in (([([1], [])], "at least one token"), ([([], [3])], "at least one token"), ([([1], [100])], "out of range"),
                       ([([1] * 60, [2] * 10)], "context length"), ([([1], [2]), ([-3], [2])], "request 1")):
        with pytest.raises(ValueError, match=what):
            m.score_many(reqs)
    assert m._lib.calls == []


def test_score_of_nothing_runs_nothing():
    lp, gr = stub_llm().score([])
    assert lp.shape == (0,) and gr.shape == (0,)


def test_entry_points_refuse_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rows = np.zeros((2, 8), np.float32)
    lp, gr = np.zeros(2), np.zeros(2, np.int32)
    assert lib.ctb_row_logprob(rows.ctypes.data_as(C.c_void_p), 2, 8, (C.c_int * 2)(1, -1), lp.ctypes.data_as(C.POINTER(C.c_double)),
                               gr.ctypes.data_as(C.POINTER(C.c_int))) == -1
