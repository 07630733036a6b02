#!/usr/bin/env python
"""What a beam search step costs: MultiLLM.beam_search against the reference's strategy replayed on this engine.
python tools/beam_search_rate.py [--steps N] [--reps 2] [--dir DIR]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, written from seed 0), in a 32-slot MultiLLM at context 512,
after a 256-token prompt (evaluated at batch size 512).  Rows:
  * beam_search at n_beams 1, 2, 4 and 8, and beam_search_many of 8 prompts at 4 beams: ms per step (MultiLLM.beam_stats, host
    clock), split into the batched eval (of the steps that evaluate no prompt), the row fetch + host selection, and the
    re-parenting launch.  A first search of the same shape warms up; the best of --reps searches is printed.
  * replay: the reference's strategy (llama.cpp:4334-4579) on one single-sequence LLM: each step evaluates the beams' common
    prefix as one chunk, then each live beam's remaining tokens as one chunk, beam after beam; the selection is ctb_beam_step.
    The host clock runs around the evals only.  Its response must equal beam_search's.
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
import beam_search_cases as B  # noqa: E402
from ctransformers_b200 import AutoModelForCausalLM, Config, MultiLLM, synth  # noqa: E402

CTX, PROMPT, N_SLOTS, BATCH = 512, 256, 32, 512


def prompts(n):
    out = []
    for s in range(n):
        ids = np.random.default_rng(100 + s).integers(259, synth.LLAMA2_7B.n_vocab, PROMPT).tolist()
        ids[0] = 1
        out.append(ids)
    return out


def device_step(lib):
    """the selection step of B.beam_search through ctb_beam_step (the library's host selection)"""
    def step(nb, beams, nxt, rows):
        n_in, nv = len(beams), len(next(r for r in rows if r is not None))
        flat = np.zeros((n_in, nv), np.float32)
        for i, r in enumerate(rows):
            if r is not None:
                flat[i] = r
        op, ot, opp, oe = (C.c_int * nb)(), (C.c_int * nb)(), (C.c_float * nb)(), (C.c_ubyte * nb)()
        n = lib.ctb_beam_step(nb, n_in, len(nxt), (C.c_float * n_in)(*[b.p for b in beams]), C.cast((C.c_ubyte * n_in)(*[b.eob for b in beams]), C.c_void_p),
                              flat.ctypes.data_as(C.POINTER(C.c_float)), nv, op, ot, opp, C.cast(oe, C.c_void_p))
        assert n > 0
        return [B.Beam(beams[op[j]].tokens + ([ot[j]] if ot[j] >= 0 else []), opp[j], bool(oe[j]), op[j], ot[j]) for j in range(n)]
    return step


def replay(llm, prompt, nb, n_predict):
    """(response, p, steps, eval seconds) of the reference's strategy on one LLM"""
    assert llm.ctransformers_llm_batch_eval((C.c_int * len(prompt))(*prompt), len(prompt), 0, BATCH, 1)
    nv = llm.vocab_size
    spent = [0.0]

    def eval_fn(tokens, n_past):
        t0 = time.perf_counter()
        assert llm.ctransformers_llm_batch_eval((C.c_int * len(tokens))(*tokens), len(tokens), n_past, BATCH, 1)
        row = np.ctypeslib.as_array(llm.ctransformers_llm_logits_data(), (nv,)).copy()
        spent[0] += time.perf_counter() - t0
        return row
    first = np.ctypeslib.as_array(llm.ctransformers_llm_logits_data(), (nv,)).copy()
    response, p, digests, _ = B.beam_search(eval_fn, len(prompt), nb, n_predict, llm.eos_token_id, first, device_step(llm._lib))
    return response, p, len(digests) - 1, spent[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--steps", type=int, default=32, help="n_predict")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    ps = prompts(8)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.dir or tmp) / "llama7b_q4_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q4_K_M", seed=0)
        m = MultiLLM(str(path), n_slots=N_SLOTS, config=Config(context_length=CTX))
        answers = {}
        for label, nb, group in [(f"n_beams {nb}", nb, ps[:1]) for nb in (1, 2, 4, 8)] + [("8 prompts x 4 beams", 4, ps)]:
            m.beam_search_many(group, nb, a.steps, batch_size=BATCH)   # warm-up
            best = None
            for _ in range(a.reps):
                res = m.beam_search_many(group, nb, a.steps, batch_size=BATCH)
                st = m.beam_stats()
                n = st["steps"] - st["prompt_steps"]   # steps that evaluated beams only
                per = [(st["eval_ms"] - st["prompt_eval_ms"]) / n, st["select_ms"] / st["steps"], st["reparent_ms"] / st["steps"]]
                if best is None or sum(per) < sum(best[0]):
                    best = (per, st)
            per, st = best
            answers[label] = res
            print(f"{label:20s} steps {st['steps']:3.0f}  eval {per[0]:7.2f}  fetch+select {per[1]:6.2f}  reparent {per[2]:6.3f}  "
                  f"= {sum(per):7.2f} ms/step  reparent {st['reparent_bytes'] / st['steps'] / 2 ** 20:6.1f} MiB/step  "
                  f"tokens {st['tokens']:.0f}  (prompt steps {st['prompt_steps']:.0f}: {st['prompt_eval_ms']:.1f} ms)", flush=True)
        del m
        llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=CTX)
        for nb in (1, 2, 4, 8):
            response, p, steps, sec = replay(llm, ps[0], nb, a.steps)
            same = (response, np.float32(p)) == (answers[f"n_beams {nb}"][0][0], np.float32(answers[f"n_beams {nb}"][0][1]))
            print(f"replay n_beams {nb}: {steps} steps, evals {1e3 * sec / max(steps, 1):7.2f} ms/step, response equal to beam_search: {same}",
                  flush=True)
            assert same
        if not a.dir:
            path.unlink()


if __name__ == "__main__":
    main()
