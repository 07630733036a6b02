"""The runs whose every-token logits rows (the reference's logits_all) are pinned by tests/golden/logits_all_runs.npz: each golden
model case of modelcases / q3k_refs / q41_q51_refs / head_dims_refs (not the 7B- / 3B-shaped ones) with its prompt at batch
sizes 8, 64 and 5 (the long-prompt cases at the one batch size of their tables), and one eval that overflows the context, so that LLM::BatchEval clamps n_past."""
import head_dims_refs as H
import modelcases
import q3k_refs as Q
import q41_q51_refs as Q1

BATCH_SIZES = (8, 64, 5)


def _table(name):
    """(arch, shape, ftype, ctx, prompt, builder, batch sizes, oracle class)"""
    if name in modelcases.CASES:
        arch, shape, ftype, ctx = modelcases.CASES[name]
        return arch, shape, ftype, ctx, modelcases.prompt_for(name), modelcases.build, BATCH_SIZES, None
    if name in H.model_cases():
        arch, shape, ftype, ctx, _, bss = H.model_cases()[name]
        return arch, shape, ftype, ctx, H.prompt_for(name), H.build_model, bss, H.OracleModel
    if name in Q.model_cases():
        arch, shape, ftype, ctx, _, bss, _ = Q.model_cases()[name]
        return arch, shape, ftype, ctx, Q.prompt_for(name), Q.build_model, bss, Q.OracleModel
    arch, shape, ftype, _, ctx, _ = Q1.model_cases()[name]
    return arch, shape, ftype, ctx, Q1.prompt_for(name), Q1.build_model, Q1.BATCH_SIZES, Q1.OracleModel


def names():
    return list(modelcases.CASES) + list(H.model_cases()) + list(Q.model_cases()) + list(Q1.model_cases())


def build(name, directory):
    return _table(name)[5](name, directory)


def n_vocab(name):
    return _table(name)[1].n_vocab


def arch(name):
    return _table(name)[0]


def ctx(name):
    return _table(name)[3]


def prompt(name):
    return _table(name)[4]


_libs = {}


def oracle_lib(tu):
    """tests/logits_all_oracle.c (the oracle plus orc_eval_all) on the oracle translation unit tu (None: the plain oracle)."""
    if tu not in _libs:
        import atexit
        import ctypes as C
        import shutil
        import subprocess
        import tempfile
        from pathlib import Path
        here = Path(__file__).resolve().parent
        d = Path(tempfile.mkdtemp(prefix="logits_all_oracle_"))
        atexit.register(shutil.rmtree, d, True)
        so = d / "liblogitsalloracle.so"
        define = [f'-DORACLE_TU="{tu}"'] if tu else []
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-mf16c", "-mavx2", "-mfma", "-ffp-contract=off", *define,
                               "-o", str(so), str(here / "logits_all_oracle.c"), "-lm"])
        o = C.CDLL(str(so))
        o.orc_eval_all.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _libs[tu] = o
    return _libs[tu]


_TU = {H: "head_dims_oracle.c", Q: "q3k_oracle.c", Q1: "q41_q51_oracle.c"}


def oracle(name, path, n_ctx=None):
    """The whole-model oracle of the case (refs.OracleModel or its per-type subclass), at its context length by default, on a
    library that also has orc_eval_all: the subclass's own oracle source with orc_eval_all appended."""
    import refs
    cls = _table(name)[7]
    n_ctx = n_ctx or ctx(name)
    if cls is None:
        saved = refs._oracle
        refs._oracle = oracle_lib(None)
        try:
            return refs.OracleModel(path, n_ctx)
        finally:
            refs._oracle = saved
    mod = next(m for m in _TU if m.OracleModel is cls)
    saved = mod._lib                 # the subclass loads its module's library through mod.oracle(), which returns mod._lib
    mod._lib = oracle_lib(_TU[mod])
    try:
        return cls(path, n_ctx)
    finally:
        mod._lib = saved


OVERFLOW = "overflow_llama_tiny_q4km"


def runs():
    """key -> (model case, [(tokens, batch_size) of each eval call, in order])."""
    out = {}
    for name in names():
        for bs in _table(name)[6]:   # (the 1100-token prompts of the long cases: one chunking, 512)
            out[f"{name}_bs{bs}"] = (name, [(prompt(name), bs)])
    # context 96: 37 prompt tokens at batch_size 8, then 80 tokens at 64: the first chunk's n_past is clamped from 37 to 32, the
    # second evaluates positions 80 .. 95
    base = "llama_tiny_q4km"
    more = modelcases.seeded_prompt(base, 81, seed=41)[1:]
    out[OVERFLOW] = (base, [(prompt(base), 8), (more, 64)])
    return out


# ------------------------------------------------------------------------------------------ float64 scores (csrc/score_gpu.cuh)
def greedy_ref(row):
    """The reference's top_k = 1 scan (block_argmax): the lowest id of the largest value; NaNs never win; id 0 when nothing
    exceeds -inf or when row[0] is NaN."""
    import numpy as np
    row = np.asarray(row, np.float32)
    v = np.where(np.isnan(row), -np.inf, row)
    if np.isnan(row[0]) or not (v > -np.inf).any():
        return 0
    return int(np.argmax(v))


def logprob_ref(rows, targets):
    """k_row_logprob in float64 numpy: (logprob, greedy) per row, with the header's rules for rows that are not all finite."""
    import numpy as np
    rows = np.atleast_2d(np.asarray(rows, np.float32))
    lp, gr = np.zeros(len(rows)), np.zeros(len(rows), np.int32)
    for r, (row, t) in enumerate(zip(rows, targets)):
        t = int(t)
        if t < 0:
            continue
        gr[r] = int(t == greedy_ref(row))
        if np.isnan(row).any():
            lp[r] = np.nan
        elif (row == np.inf).any():
            lp[r] = -np.log(float((row == np.inf).sum())) if row[t] == np.inf else -np.inf
        elif (row == -np.inf).all():
            lp[r] = np.nan
        else:
            m = np.float64(row.max())
            lp[r] = (np.float64(row[t]) - m) - np.log(np.sum(np.exp(row.astype(np.float64) - m)))
    return lp, gr


def oracle_rows(model, tokens, batch_size, n_ctx):
    """orc_eval_all, chunked and clamped as LLM::BatchEval: the row block of each chunk."""
    import numpy as np
    o = model.o   # (a model from oracle())
    bs, blocks = min(n_ctx, batch_size), []
    for start in range(0, len(tokens), bs):
        chunk = np.array(tokens[start:start + bs], np.int32)
        past = min(n_ctx - len(chunk), model.n_past)
        rows = np.zeros((len(chunk), model.n_vocab), np.float32)
        assert o.orc_eval_all(model.m, chunk.ctypes.data, len(chunk), past, rows.ctypes.data, model.embd.ctypes.data) == 0
        model.n_past += len(chunk)
        blocks.append(rows)
    return blocks


def chunk_sizes(n, batch_size, n_ctx):
    bs = min(n_ctx, batch_size)
    return [min(bs, n - s) for s in range(0, n, bs)]


def digests(rows, sizes):
    import hashlib
    import numpy as np
    out, at = [], 0
    for k in sizes:
        out.append(hashlib.sha256(np.ascontiguousarray(rows[at:at + k], np.float32).tobytes()).hexdigest())
        at += k
    return out


def golden():
    import numpy as np
    import refs
    return np.load(refs.GOLD / "logits_all_runs.npz")
