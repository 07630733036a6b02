#!/usr/bin/env python
"""What choosing the next token costs a MultiLLM step: per-slot sampling against MultiLLM.sample_many.
python tools/multi_sample_rate.py [--parent-lib PATH] [--steps N] [--slots 1,8,32] [--reps 2]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, written from seed 0), in a 32-slot handle at context 512: S slots
evaluate 256-token prompts together, then lockstep steps run.  A step is one eval of one token per slot (ctb_multi_eval) and the
draw of every slot; the host clock runs around both, and each ends by synchronising the engine stream.  Two settings: the config
defaults (top_k 40, top_p 0.95, temperature 0.8, repetition_penalty 1.1, last_n_tokens 64) and greedy (top_k 1, no penalty).
Slot s draws with seed 1000 * step + s.

Columns: `per-slot` draws with one ctb_multi_sample call per slot, as MultiLLM.sample did in a loop; `sample_many` draws all slots
with one call.  --parent-lib runs the per-slot loop on another build of the library too (the commit before sample_many existed,
whose ctb_multi_sample copied each slot's logits to the host and sorted them there); the builds alternate, --reps times, in
one process, and their tokens must be equal.  Also printed: the GPU, its power limit and maximum SM clock."""
import argparse
import ctypes as C
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import Config, MultiLLM, synth  # noqa: E402

CTX, PROMPT, N_SLOTS, WARMUP = 512, 256, 32, 3
SETTINGS = {"default": dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1, last_n_tokens=64),
            "greedy": dict(top_k=1, top_p=0.95, temperature=0.8, repetition_penalty=1.0, last_n_tokens=64)}


def prompts(n_slots):
    out = []
    for s in range(n_slots):
        ids = np.random.default_rng(100 + s).integers(259, synth.LLAMA2_7B.n_vocab, PROMPT).tolist()
        ids[0] = 1
        out.append(ids)
    return out


def per_slot(m, slots, seeds, st):
    """One ctb_multi_sample per slot (MultiLLM.sample's call, which a library without sample_many also has)."""
    out = []
    for s, seed in zip(slots, seeds):
        recent = m.context(s)[-st["last_n_tokens"]:]
        t = m._lib.ctb_multi_sample(m._m, s, (C.c_int * max(len(recent), 1))(*recent), len(recent), st["top_k"], st["top_p"], st["temperature"],
                                    st["repetition_penalty"], seed)
        assert t >= 0
        out.append(t)
    return out


def many(m, slots, seeds, st):
    return m.sample_many(slots, seed=seeds, **st)


def run(m, ps, steps, st, draw):
    """Lockstep steps of len(ps) slots; returns eval ms / step, sampling ms / step and every slot's tokens."""
    S = len(ps)
    for s in range(S):
        m.reset(s)
    m.eval(dict(enumerate(ps)), batch_size=512)
    slots = list(range(S))
    toks = [draw(m, slots, [s for s in slots], st)]
    t_eval = t_samp = 0.0
    for i in range(WARMUP + steps):
        t0 = time.perf_counter()
        m.eval({s: [t] for s, t in enumerate(toks[-1])})
        t1 = time.perf_counter()
        toks.append(draw(m, slots, [1000 * (i + 1) + s for s in slots], st))
        t2 = time.perf_counter()
        if i >= WARMUP:
            t_eval += t1 - t0
            t_samp += t2 - t1
    return 1e3 * t_eval / steps, 1e3 * t_samp / steps, toks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--parent-lib")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--slots", default="1,8,32")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    slots = [int(x) for x in a.slots.split(",")]
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    builds = [("this", None, [("per-slot", per_slot), ("sample_many", many)])]
    if a.parent_lib:
        builds.insert(0, ("parent", a.parent_lib, [("per-slot", per_slot)]))
    ps = prompts(N_SLOTS)
    results, tokens = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.dir or tmp) / "llama7b_q4_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q4_K_M", seed=0)
        for rep in range(a.reps):
            for bname, lib, draws in builds:
                m = MultiLLM(str(path), n_slots=N_SLOTS, config=Config(context_length=CTX), lib=lib)
                for S in slots:
                    for sname, st in SETTINGS.items():
                        for dname, draw in draws:
                            ev, sm, toks = run(m, ps[:S], a.steps, st, draw)
                            key = (S, sname, f"{bname} {dname}")
                            results.setdefault(key, []).append((ev, sm))
                            want = tokens.setdefault((S, sname), toks)
                            assert toks == want, f"{key}: tokens differ from the first run of these settings"
                            print(f"rep {rep} S={S:2d} {sname:7s} {bname} {dname:11s}: eval {ev:7.3f} ms  sampling {sm:7.3f} ms  "
                                  f"step {ev + sm:7.3f} ms", flush=True)
                del m
        if not a.dir:
            path.unlink()
    print("\nbest of the reps, ms per step (eval + sampling of all slots; sampling alone in brackets)")
    for (S, sname, name), v in sorted(results.items()):
        ev, sm = min(v, key=lambda x: x[0] + x[1])
        print(f"S={S:2d} {sname:7s} {name:20s} {ev + sm:8.3f}  ({sm:7.3f})")


if __name__ == "__main__":
    main()
