"""The norm prologue of every mat-vec kernel against the oracle, bit for bit, on rows where the order of the fp64 sums reaches
the float result (refs.norm_order_rows).  The kernels add the terms in another order than the reference; stage_activation
(csrc/matvec.cuh norm_stat) proves when that order gives the reference's float and otherwise adds them in element order.
A kernel that trusted its own order fails here: test_norm_order.py shows that order changing every one of these rows."""
import ctypes as C

import numpy as np
import pytest

import modelcases
import refs
from conftest import ptr
from refs import Q4_K
from test_norm_order import KS, _oracle_norm
from test_ops_gpu import STORE, _pf_expected, _pf_run, _same_bits

pytestmark = pytest.mark.gpu

PATHS = {0: "k_matvec", 1: "k_step"}
PB_NT = 256   # k_pstep's prologue threads (prefill.cuh PB_NT)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("path", list(PATHS), ids=list(PATHS.values()))
def test_norm_paths_planted_rows(lib, path, mode, k):
    if path == 1 and k % 256:
        pytest.skip("the step kernel takes widths that are multiples of 256")
    rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
    want = _oracle_norm(mode, rows, w, b, refs.NORM_ORDER_EPS)
    got = np.zeros_like(rows)
    for i in range(rows.shape[0]):
        assert lib.ctb_norm_path(path, mode, ptr(rows[i]), ptr(w), ptr(b) if mode == 2 else None, ptr(got[i]), k, refs.NORM_ORDER_EPS) == 0
    bad = (got.view(np.uint32) != want.view(np.uint32)).any(axis=1)
    assert not bad.any(), f"rows {np.flatnonzero(bad).tolist()} of {rows.shape[0]} differ"


def test_norm_path_refuses_what_it_cannot_take(lib):
    x = np.ones(384, np.float32)
    y = np.zeros_like(x)
    assert lib.ctb_norm_path(1, 1, ptr(x), ptr(x), None, ptr(y), 384, 1e-5) == -1
    assert lib.ctb_norm_path(2, 1, ptr(x), ptr(x), None, ptr(y), 256, 1e-5) == -1
    assert lib.ctb_norm_path(0, 0, ptr(x), ptr(x), None, ptr(y), 256, 1e-5) == -1


@pytest.mark.parametrize("mode,k", [(1, 4096), (2, 4608)])
def test_prefill_mul_mat_planted_rows(lib, mode, k):
    """The batched prefill's QUANT phase normalises each token row with k_pstep's own CTA size.  Planted rows sit among ordinary
    ones in the first full launch and in the short last one (70 tokens = 32 + 32 + 6).  Expected values as for
    test_ops_gpu.test_prefill_mul_mat_shapes."""
    rows, w, _ = refs.norm_order_rows(mode, k, seed=k + 10 * mode)
    b = np.zeros(k, np.float32)   # no bias: a LayerNorm row's changed mean then moves every element of the blocks without x0
    rng = np.random.default_rng(mode)
    x = (rng.standard_normal((70, k)) * 2).astype(np.float32)
    at = [0, 5, 17, 31, 40, 64, 66, 69]                    # 4 in the first full launch, 3 in the short last one
    x[at] = np.resize(rows, (len(at), k))                  # (RMSNorm has 4 planted rows: each is used twice)
    segs = [(Q4_K, 48, STORE)]
    ws = [np.ascontiguousarray(refs.reference_quantized_blocks(Q4_K, k, 48, seed=mode))]
    res = np.zeros((70, 48), np.float32)
    want, _ = _pf_expected(segs, ws, k, x, None, mode, w, b, res, res)
    # the rows the kernels' own order would produce change the product: the comparison below can see the difference
    y_k, _ = refs.norm_emulated(mode, x, w, b, 1e-5, lambda t: refs.kernel_order_sum(t, PB_NT))
    y_k = np.ascontiguousarray(y_k)
    wrong = np.zeros_like(want)
    assert refs.oracle().orc_mul_mat(Q4_K, ptr(ws[0]), ptr(y_k), ptr(wrong), k, 48, 70) == 0
    assert (wrong != want).any(axis=1)[at].all()
    for n in (1, 33, 70):
        rc, got, _ = _pf_run(lib, segs, ws, k, x[:n], None, mode, w, b, res[:n], res[:n])
        assert rc == 0
        try:
            _same_bits(got, want[:n])
        except AssertionError as e:
            raise AssertionError(f"n_tok {n}: {e}") from None


# ---- whole models: planted embedding rows reach the first layer's norm through the engine's own wiring (model eps, LayerNorm
# weight and bias, which kernel each path takes)
@pytest.fixture(scope="module")
def norm_model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("norm_order_models")


_oracle_runs = {}


def _paths(llm):
    from test_long_context_gpu import PATH_FIELDS
    out = (C.c_int * len(PATH_FIELDS))()
    assert llm.ctb_llm_paths(out, len(PATH_FIELDS)) == len(PATH_FIELDS)
    return dict(zip(PATH_FIELDS, out))


@pytest.mark.parametrize("prefill", [True, False], ids=["prefill", "no-prefill"])
@pytest.mark.parametrize("name", list(modelcases.NORM_ORDER_MODELS))
def test_planted_tokens_whole_model(name, prefill, norm_model_dir, monkeypatch):
    """Logits and embeddings after the prompt and after every decode step, and the greedy tokens: bit for bit the oracle's and the
    reference's (digests in reference_runs.npz).  With CTB_NO_PREFILL=1 the prompt runs through the single-token kernel too."""
    from ctransformers_b200 import AutoModelForCausalLM
    if not prefill:
        monkeypatch.setenv("CTB_NO_PREFILL", "1")
    path, ctx = modelcases.build_norm_order(name, norm_model_dir)
    if name not in _oracle_runs:
        _oracle_runs[name] = modelcases.norm_order_oracle_run(refs.OracleModel(path, ctx), name)
    o_states, o_toks = _oracle_runs[name]
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    states, toks = modelcases.norm_order_llm_run(llm, name)
    got = _paths(llm)
    # Q4_0 weights are no step-kernel type: that model's mat-vecs run k_matvec, and it has no batched prefill.  The greedy steps
    # may be served by the engine's look-ahead, so only the planted decode steps count towards single_steps for sure.
    kquant = modelcases.CASES[name][2] != "Q4_0"
    assert got["fused"] == 1 and got["prefill_ok"] == int(kquant and prefill), got
    assert got["prefill_launches"] == (2 if kquant and prefill else 0), got   # 40 tokens: one full launch and a short one
    assert got["single_steps"] >= len(modelcases.NORM_ORDER_PLANTED) + (0 if kquant and prefill else modelcases.NORM_ORDER_PROMPT), got
    gold = refs.golden_runs()
    for i, ((lg, em), (o_lg, o_em)) in enumerate(zip(states, o_states)):
        _same_bits(lg, o_lg)
        _same_bits(em, o_em)
        assert refs.digest(lg) == str(gold[f"norm_{name}_{i}_logits"]), f"state {i}: logits are not the reference's bits"
        assert refs.digest(em) == str(gold[f"norm_{name}_{i}_embd"]), f"state {i}: embeddings are not the reference's bits"
    assert toks == o_toks == gold[f"norm_{name}_tokens"].tolist()
