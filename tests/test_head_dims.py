"""Head sizes other than 64 / 128 on the CPU: the oracle's whole-model runs of the head_dims_refs cases equal the reference's
stored results (golden/head_dims_runs.npz) at the same chunkings, which pins the oracle's K·q tail (elements
head_dim & ~31 .. head_dim-1, added one by one in double after the lane reduction) against the real reference; and the
stored results tell that tail from the forms the reference does not use."""
import numpy as np
import pytest

import head_dims_refs as H
import modelcases
import refs

RUNS = [(name, bs) for name, case in H.model_cases().items() for bs in case[5]]


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("head_dims_models")


def results(run):
    first_logits, first_embd, toks, last_logits, _ = run
    return {"tokens": toks, "first_logits": refs.digest(first_logits), "first_embd": refs.digest(first_embd),
            "last_logits": refs.digest(last_logits)}


def stored(key):
    gold = H.golden_runs()
    return {"tokens": gold[f"{key}_tokens"].tolist(), **{k: str(gold[f"{key}_{k}"]) for k in ("first_logits", "first_embd", "last_logits")}}


@pytest.mark.parametrize("name,bs", RUNS, ids=[f"{n}-bs{b}" for n, b in RUNS])
def test_whole_model_oracle_matches_reference(name, bs, model_dir):
    path, ctx = H.build_model(name, model_dir)
    run = modelcases.oracle_greedy(H.OracleModel(path, ctx), H.prompt_for(name), H.N_NEW, bs)
    assert results(run) == stored(f"{name}_bs{bs}")


@pytest.mark.parametrize("variant", [H.TAIL_FP32, H.TAIL_IN_LANES], ids=["tail-fp32", "tail-in-lanes"])
def test_other_tails_give_other_bits(variant, model_dir):
    """The K·q tail summed in fp32, or folded into the SIMD lanes, changes at least one stored result of the hd 100 and
    hd 80 cases (tails of 4 and 16 elements)."""
    changed = []
    for name in ("llama_hd100_q4_0", "llama_hd80_q4km_gqa"):
        path, ctx = H.build_model(name, model_dir)
        run = modelcases.oracle_greedy(H.OracleModel(path, ctx, variant), H.prompt_for(name), H.N_NEW, 8)
        got, want = results(run), stored(f"{name}_bs8")
        changed += [f"{name}:{k}" for k in want if got[k] != want[k]]
    assert changed, "the stored results do not tell this tail from the reference's"


def test_model_cases_have_the_promised_head_sizes():
    sizes = {name: case[1].n_embd // case[1].n_head for name, case in H.all_cases().items()}
    assert sizes == {"llama_hd100_q4_0": 100, "llama_hd100_gqa_q4_0": 100, "llama_hd80_q4km_gqa": 80, "llama_hd96_q5km": 96,
                     "falcon_hd96_q5km_mqa": 96, "llama_hd80_long": 80, "openllama3b_q4_0": 100}
