"""The last step of a token, host side: the plain numpy references the device pick and the device top-k are checked against
(test_pick_gpu.py), and the adversarial logit vectors they are checked on.  Here the references are pinned to the compiled host
sampler, which host_logic.npz pins to the reference: with top_k = 1 (and no penalty, top_p 1, temperature 1) ctb_sample must
pick what the reference's sequential scan picks on every vector, NaN and infinities included."""
import ctypes as C

import numpy as np
import pytest

F32 = np.float32
FMAX = np.finfo(F32).max
TINY = np.finfo(F32).smallest_subnormal
ARGMAX_NT, STEP_NT = 1024, 320   # threads of k_argmax and of the step kernel's PH_PICK phase (attention.cuh, stream.cuh ST_NT)

# warp and block sweeps of both builds, the step kernel's 4-deep unroll (4 * 320 = 1280), and real vocabularies
SIZES = [1, 2, 31, 32, 33, 319, 320, 321, 1023, 1024, 1025, 1279, 1280, 1281, 32000, 32001, 50257, 65024, 151936, 256000]


# ------------------------------------------------------------------------------------------------------------- references
def scan_pick(x):
    """The reference's top_k = 1 (std::partial_sort of one element): start at element 0, move on strictly greater only."""
    cur = 0
    for i in range(1, len(x)):
        if x[i] > x[cur]:
            cur = i
    return cur


def ref_pick(x):
    """scan_pick without the Python loop.  From a NaN at 0 nothing is greater; otherwise NaNs never win, and the first largest of
    the rest does (the value at the cursor only rises, so it stops at the first occurrence of the largest)."""
    if np.isnan(x[0]):
        return 0
    m = np.nanmax(x)
    return int(np.flatnonzero(x == m)[0])


def ref_ties(x, pick):
    """k_argmax's second output: how many logits equal the picked one (0 for a NaN)."""
    return int((x == x[pick]).sum())


def penalise(x, last, penalty):
    """The repetition penalty (llama.cpp:4025-4055) in float32: once per id of `last` inside [0, n), x * p for x <= 0, else x / p."""
    y = np.array(x, F32, copy=True)
    last = np.asarray(last, np.int64)
    if len(last) == 0 or penalty == 1.0:
        return y
    ids = np.unique(last[(last >= 0) & (last < len(y))])
    v = y[ids]
    with np.errstate(invalid="ignore", over="ignore"):   # (FLT_MAX * 1.3 is inf, as in float32 on the device and the host)
        y[ids] = np.where(v <= 0, v * F32(penalty), v / F32(penalty)).astype(F32)
    return y


def ref_topk(y, k):
    """Ids of every penalised logit >= the k-th largest (k capped at n), or None when some logit is NaN (no order: the host
    decides)."""
    if np.isnan(y).any():
        return None
    k = min(k, len(y))
    kth = np.partition(y, len(y) - k)[len(y) - k]
    return np.flatnonzero(y >= kth)


def device_answers(x, last, top_k, penalty):
    """Whether the lazy chain of ctransformers_llm_sample can answer on the device: the greedy shortcut on a unique arg-max, or a
    device top-k cut of exactly k distinct logits.  Everything else goes to the host sampler."""
    if top_k == 1 and (penalty == 1.0 or len(last) <= 0):
        p = ref_pick(x)
        if ref_ties(x, p) == 1:
            return True
    if len(last) > 256 or top_k < 1 or top_k > 128:
        return False
    y = penalise(x, last, penalty)
    ids = ref_topk(y, top_k)
    if ids is None or len(ids) != min(top_k, len(x)):
        return False
    return len(np.unique(y[ids])) == len(ids)   # (-0.0 and +0.0 count as equal, as they do for the host's ==)


# ------------------------------------------------------------------------------------------------------------- vectors
def _normal(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(F32)


def _with(x, at, v):
    x = x.copy()
    x[[a for a in at if a < len(x)]] = v
    return x


def boundary_ids(n):
    """Lane, warp and block boundaries of both builds, and the first element of each one's ragged last sweep."""
    ids = {0, n - 1, 1, 31, 32, 63, 64, 319, 320, 639, 640, 1023, 1024, 1279, 1280, 4 * STEP_NT + 31, n - n % STEP_NT, n - n % ARGMAX_NT,
           n - n % (4 * STEP_NT)}
    return sorted(i for i in ids if 0 <= i < n)


def zero_threshold(n, k, neg_low, seed=0):
    """k - 1 positive logits, everything else <= -1 but a -0.0 and a +0.0: the k-th largest is a zero with an equal one beside
    it.  neg_low puts the -0.0 at the lower id of the two."""
    rng = np.random.default_rng(seed + n + k)
    x = (-1.0 - np.abs(rng.standard_normal(n))).astype(F32)
    ids = rng.permutation(n)
    x[ids[: k - 1]] = (1.0 + np.abs(rng.standard_normal(k - 1))).astype(F32)
    a, b = sorted(ids[k - 1: k + 1].tolist())
    x[a], x[b] = (F32(-0.0), F32(0.0)) if neg_low else (F32(0.0), F32(-0.0))
    return x


def vectors(n):
    """(name, logits) pairs: the cases where a block-wide arg-max or a radix select goes wrong."""
    x = _normal(n, n)
    low = np.full(n, -5.0, F32)
    out = [("normal", x)]
    for i in boundary_ids(n):
        out.append((f"max_at_{i}", _with(low, [i], 3.0)))
    # equal maxima: one thread (ids NT apart), one warp (neighbouring lanes), across warps, and where the higher id sits in a lower
    # thread (thread 0 holds NT, thread 1 holds 1: the lower id must win the shuffle)
    for nt in (STEP_NT, ARGMAX_NT):
        if n > nt + 5:
            out.append((f"tie_thread_{nt}", _with(low, [5, nt + 5], 3.0)))
            out.append((f"tie_lane_order_{nt}", _with(low, [1, nt], 3.0)))
    if n > 7:
        out.append(("tie_warp", _with(low, [6, 7], 3.0)))
    if n > 700:
        out.append(("tie_across_warps", _with(low, [37, 700, n - 1], 3.0)))
    out.append(("tie_first_last", _with(low, [0, n - 1], 3.0)))
    out += [("all_equal", np.full(n, 0.5, F32)), ("all_neg_inf", np.full(n, -np.inf, F32)),
            ("neg_inf_but_one", _with(np.full(n, -np.inf, F32), [n // 2], -7.0)),
            ("pos_infs", _with(x, [n // 3, n // 2, n - 1], np.inf)),
            ("neg_inf_and_nan", _with(np.full(n, -np.inf, F32), [n - 1], np.nan))]
    if n >= 2:
        for neg_low in (True, False):
            a, b = (n // 3, n - 1) if n > 2 else (0, 1)
            z = _with(low, [a], F32(-0.0) if neg_low else F32(0.0))
            z[b] = F32(0.0) if neg_low else F32(-0.0)
            out.append((f"zero_max_neg_{'low' if neg_low else 'high'}", z))
    big = _with(np.full(n, -FMAX, F32), [n // 2], FMAX)
    sub = (np.random.default_rng(n + 1).integers(-8, 9, n) * TINY).astype(F32)
    out += [("flt_max", big), ("subnormals", sub), ("subnormals_neg_flt_max", _with(sub, [0, n - 1], -FMAX))]
    out += [("nan_at_0", _with(x, [0], np.nan)), ("nan_at_0_rest_neg_inf", _with(np.full(n, -np.inf, F32), [0], np.nan)),
            ("nan_elsewhere", _with(x, [1, n // 2, n - 1], np.nan)), ("all_nan", np.full(n, np.nan, F32))]
    out.append(("grid", (np.floor(x * 2) / 2).astype(F32)))          # many equal logits: thresholds tie
    out.append(("coarse_grid", np.floor(x).astype(F32)))             # tie counts far above k and above 256
    return out


def sampler_vectors(n, k):
    """vectors(n) plus the two signed-zero threshold cases for this k."""
    out = vectors(n)
    if 2 <= k <= n - 2:
        out += [("zero_threshold_neg_low", zero_threshold(n, k, True)), ("zero_threshold_neg_high", zero_threshold(n, k, False))]
    return out


# ------------------------------------------------------------------------------------------------------------- tests
def test_vectorised_pick_is_the_scan():
    for n in SIZES[:14] + [32000]:
        for name, x in vectors(n):
            assert ref_pick(x) == scan_pick(x), (n, name)


@pytest.mark.parametrize("n", SIZES)
def test_host_sampler_top1_is_the_scan(lib, n):
    """ctb_sample with top_k = 1 is std::partial_sort over all candidates: the scan, even where NaN breaks the strict weak order."""
    for name, x in vectors(n):
        x = np.ascontiguousarray(x, F32)
        got = lib.ctb_sample(x.ctypes.data_as(C.POINTER(C.c_float)), n, None, 0, 1, 1.0, 1.0, 1.0, 0)
        assert got == ref_pick(x), (name, got, ref_pick(x))


def test_signed_zeros_at_the_threshold_are_a_tie():
    """Why sg_key maps -0.0 to +0.0: the host's comparator sees the two zeros at this threshold as equal, so the cut of 4 holds 5
    logits and only the host's sort may choose among them."""
    x = np.array([3, 2, 1, -0.0, 0.0, -1, -2, -3], F32)
    assert ref_topk(x, 4).tolist() == [0, 1, 2, 3, 4]
    assert not device_answers(x, [], 4, 1.0)


def test_penalty_reference():
    x = np.array([2.2, -1.0, 0.0, -0.0, 3.0], F32)
    y = penalise(x, [0, 0, 1, 2, 3, -1, 5, 99], 1.1)
    assert y[0] == F32(F32(2.2) / F32(1.1)) and y[1] == F32(-1.0) * F32(1.1) and y[4] == F32(3.0)
    assert y[2] == 0 and np.signbit(y[3]) and not np.signbit(y[2])
    assert (penalise(x, [0], 1.0) == x).all() and (penalise(x, [], 1.3) == x).all()
