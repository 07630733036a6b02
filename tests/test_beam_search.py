"""CPU checks of beam search: the Python restatement of the reference's llama_beam_search (tests/beam_search_cases.py), run on the
oracle's logits with the reference's own chunks, reproduces every callback state, response and final p the reference produced
(tests/golden/beam_search_runs.npz); one beam is greedy decoding."""
import numpy as np
import pytest

import beam_search_cases as B
import modelcases
import refs


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("beam_models")


def golden():
    return np.load(refs.GOLD / "beam_search_runs.npz")


def oracle_search(name, prompt, n_beams, n_predict, model_dir):
    """The restatement on the oracle: the prompt in chunks of B.BATCH_SIZE, then one oracle eval per chunk the reference evaluates."""
    path, ctx = B.build(name, model_dir)
    model = B.oracle(name, path, ctx)
    model.eval(prompt, batch_size=B.BATCH_SIZE)

    def eval_fn(tokens, n_past):
        model.n_past = n_past
        return model.eval(tokens, batch_size=len(tokens)).copy()
    return B.beam_search(eval_fn, len(prompt), n_beams, n_predict, B.eos_of(name), model.logits.copy())


@pytest.mark.parametrize("key", list(B.cases()))
def test_restatement_on_oracle_matches_reference(key, model_dir):
    name, prompt, nb, n_predict = B.cases()[key]
    response, p, states, _ = oracle_search(name, prompt, nb, n_predict, model_dir)
    gold = golden()
    assert states == gold[f"{key}_states"].tolist()
    assert response == gold[f"{key}_response"].tolist()
    assert B.p_bits(p) == int(gold[f"{key}_p"][0])


def test_small_vocabulary_cases_reach_eos():
    """EOS reaches the beams: some runs end on an eob top beam before n_predict, with EOS as their last token."""
    gold = golden()
    ended = [k for k in B.cases() if k.startswith(B.SMALL) and 0 < len(gold[f"{k}_response"]) < B.N_PREDICT
             and gold[f"{k}_response"][-1] == B.eos_of(B.SMALL)]
    assert len(ended) >= 3, ended


@pytest.mark.parametrize("name", [n for n in B.MODELS if n in modelcases.CASES])
def test_one_beam_is_greedy(name):
    """n_beams 1 gives the greedy tokens of the model's golden run (model_<name>.npz, 24 steps), up to the first EOS."""
    tokens = np.load(refs.GOLD / f"model_{name}.npz")["tokens"].tolist()
    eos = B.eos_of(name)
    if eos in tokens:
        tokens = tokens[:tokens.index(eos) + 1]
    response = golden()[f"{name}_b1_response"].tolist()
    n = min(len(tokens), len(response))
    assert n >= min(len(tokens), 24) and response[:n] == tokens[:n]


def test_heap_algorithms_are_libstdcxx_array_order():
    """make_heap / push_heap / pop_heap of the restatement leave libstdc++'s array order (values from a g++ -O2 run of the same
    calls with std::greater<int>)."""
    comp = lambda a, b: a > b
    a = [5, 3, 8, 1, 9, 2, 7]
    B.make_heap(a, comp)
    assert a == [1, 3, 2, 5, 9, 8, 7]
    B.pop_heap(a, comp)
    assert a == [2, 3, 7, 5, 9, 8, 1]
    a[-1] = 4
    B.push_heap(a, comp)
    assert a == [2, 3, 4, 5, 9, 8, 7]
    b = [4, 4, 2, 9, 0, 6, 6, 1, 3, 3, 8, 5]   # an even length: _adjust_heap's last single child
    B.make_heap(b, comp)
    assert b == [0, 1, 2, 3, 3, 5, 6, 9, 4, 4, 8, 6]
    B.pop_heap(b, comp)
    assert b == [1, 3, 2, 3, 4, 5, 6, 9, 4, 6, 8, 0]
