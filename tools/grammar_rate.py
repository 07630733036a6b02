#!/usr/bin/env python
"""What a grammar costs a sampling step.  python tools/grammar_rate.py [--steps N] [--reps R] [--file GGUF]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, vocabulary 32000, written from seed 0, or the one --file names)
with the JSON grammar of
tests/grammar_cases.py, in three states: structural (after `{`), string (after `{"k`) and number (after `{"k":1`).

  k_grammar_mask       the kernel alone, from torch.profiler's CUDA activity: 1 row (LLM.grammar_mask) and 32 rows (one
                       MultiLLM.sample_many with a state for each of 32 slots)
  mask call            LLM.grammar_mask end to end on the host clock (upload, kernel, copy back, synchronise)
  host mask            the host code over the same state and vocabulary (ctb_grammar_mask_pieces)
  reference mask       the reference's own llama_sample_grammar on the host (oracle/_ref/libctransformers_ref.so, where built)
  LLM step             eval of one token + LLM.sample, with and without the grammar (the state stays as given)
  MultiLLM sample_many 32 slots, with a state per slot and without
Also printed: the GPU, its power limit and maximum SM clock."""
import argparse
import ctypes as C
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from ctransformers_b200 import Config, Grammar, LLM, MultiLLM, synth  # noqa: E402
import grammar_cases as G  # noqa: E402

CTX, PROMPT, N_SLOTS = 512, 256, 32
STATES = {"structural": b"{", "string": b'{"k', "number": b'{"k":1'}
DEFAULT = dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1, last_n_tokens=64)


def prompt(seed):
    ids = np.random.default_rng(seed).integers(259, synth.LLAMA2_7B.n_vocab, PROMPT).tolist()
    ids[0] = 1
    return ids


def byte_tokens(piece):
    return [3 + b for b in piece]   # the SPM vocabulary's <0xNN> tokens


def state_for(g, model, piece):
    s = g.start()
    for t in byte_tokens(piece):
        s.accept(model, t)
    return s


def kernel_ms(fn, reps):
    """mean device time of k_grammar_mask over reps calls of fn, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    times = [e.device_time_total / e.count for e in prof.key_averages() if "k_grammar_mask" in e.key and e.count]
    return times[0] / 1e3 if times else float("nan")


def wall_ms(fn, reps):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return 1e3 * (time.perf_counter() - t0) / reps


def reference_mask(path, g, reps):
    """llama_sample_grammar of the reference on the host over 32000 candidates, per state: ms per call ({} without oracle/_ref).
    The grammar is llama_grammar_init over g's rules (equal to the reference parser's, tests/test_grammar.py), advanced with
    llama_grammar_accept_token over the same byte tokens."""
    if not (ROOT / "oracle" / "_ref" / "libctransformers_ref.so").exists():
        return {}
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    import make_golden_grammar as MG
    r = MG.reference()
    r.llama_grammar_init.restype = C.c_void_p
    r.llama_grammar_init.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t]
    r.llama_grammar_free.argtypes = [C.c_void_p]
    r.llama_grammar_accept_token.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    r.llama_sample_grammar.argtypes = [C.c_void_p, C.POINTER(MG.TokenDataArray), C.c_void_p]
    n_vocab = synth.LLAMA2_7B.n_vocab
    ref = MG.RefContext(r, path, 64, n_vocab)
    rules = g.rules
    off = np.concatenate([[0], np.cumsum([len(x) for x in rules])]).astype(np.int32)
    elems = np.array([e for x in rules for e in x], np.uint32)
    template = (MG.TokenData * n_vocab)(*[MG.TokenData(i, 0.0, 0.0) for i in range(n_vocab)])
    work = (MG.TokenData * n_vocab)()
    out = {}
    for name, piece in STATES.items():
        arrays, ptrs = MG.ref_grammar(r, off, elems)
        gram = r.llama_grammar_init(ptrs, len(arrays), g.symbol_ids["root"])
        for t in byte_tokens(piece):
            r.llama_grammar_accept_token(ref.ctx, gram, t)
        t_all = 0.0
        for _ in range(reps):
            C.memmove(work, template, C.sizeof(template))
            arr = MG.TokenDataArray(work, n_vocab, False)
            t0 = time.perf_counter()
            r.llama_sample_grammar(ref.ctx, C.byref(arr), gram)
            t_all += time.perf_counter() - t0
        out[name] = 1e3 * t_all / reps
        r.llama_grammar_free(gram)
    ref.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--file", help="an existing 7B-shaped Q4_K_M file (bench.py's); by default one is written to a temporary directory")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    g = Grammar(G.JSON)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.file) if a.file else Path(tmp) / "llama7b_q4_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q4_K_M", seed=0)
        pieces = G.pieces_of(path)
        off = (C.c_int * (len(pieces) + 1))(*np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(int).tolist())
        blob = b"".join(pieces)
        out = np.zeros(len(pieces), np.uint8)
        rows = {}
        llm = LLM(str(path), config=Config(context_length=CTX))
        states = {k: state_for(g, llm, v) for k, v in STATES.items()}
        for name, s in states.items():
            r = rows.setdefault(name, {})
            r["allowed"] = int(llm.grammar_mask(s).sum())
            r["kernel 1 row"] = kernel_ms(lambda: llm.grammar_mask(s), a.reps)
            r["mask call"] = wall_ms(lambda: llm.grammar_mask(s), a.reps)
            r["host mask"] = wall_ms(lambda: llm._lib.ctb_grammar_mask_pieces(s._s, len(pieces), off, blob, 2, out.ctypes.data), 3)
        # LLM step: eval one token + sample, with and without the grammar
        llm.eval(prompt(1), batch_size=512)

        def steps(grammar):
            llm.load_state(saved)
            tok = llm.sample(seed=0, grammar=grammar, **DEFAULT)
            t0 = time.perf_counter()
            for i in range(a.steps):
                llm.eval([tok])
                tok = llm.sample(seed=i, grammar=grammar, **DEFAULT)
            return 1e3 * (time.perf_counter() - t0) / a.steps
        saved = llm.save_state()
        steps(None)
        step_plain = min(steps(None) for _ in range(2))
        for name, s in states.items():
            steps(s)
            rows[name]["LLM step"] = min(steps(s) for _ in range(2))
        print(f"LLM step without grammar: {step_plain:.3f} ms", flush=True)
        del llm
        m = MultiLLM(str(path), n_slots=N_SLOTS, config=Config(context_length=CTX))
        m.eval({s: prompt(100 + s) for s in range(N_SLOTS)}, batch_size=512)
        slots = list(range(N_SLOTS))
        seeds = list(range(N_SLOTS))
        plain = wall_ms(lambda: m.sample_many(slots, seed=seeds, **DEFAULT), a.reps)
        print(f"MultiLLM sample_many, {N_SLOTS} slots, without grammar: {plain:.3f} ms", flush=True)
        for name in states:
            sts = [state_for(g, m, STATES[name]) for _ in slots]
            rows[name]["kernel 32 rows"] = kernel_ms(lambda: m.sample_many(slots, seed=seeds, grammars=sts, **DEFAULT), a.reps)
            rows[name]["sample_many 32"] = wall_ms(lambda: m.sample_many(slots, seed=seeds, grammars=sts, **DEFAULT), a.reps)
        print(f"grammar paths of the MultiLLM: {m.grammar_paths()}")
        del m
        for name, ms in reference_mask(path, g, 5).items():
            rows[name]["reference mask"] = ms
        if not a.file:
            path.unlink()
    cols = ["allowed", "kernel 1 row", "kernel 32 rows", "mask call", "host mask", "reference mask", "LLM step", "sample_many 32"]
    print("\nms (allowed: tokens the state allows of 32000)")
    print(f"{'state':12s}" + "".join(f"{c:>16s}" for c in cols))
    for name, r in rows.items():
        cell = lambda v: f"{'-':>16s}" if v is None else f"{v:16.3f}" if isinstance(v, float) else f"{v:16d}"
        print(f"{name:12s}" + "".join(cell(r.get(c)) for c in cols))


if __name__ == "__main__":
    main()
