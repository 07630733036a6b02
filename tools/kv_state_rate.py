#!/usr/bin/env python
"""What sequence states cost against evaluating the prompt again: python tools/kv_state_rate.py [--dir DIR] [--reps N]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, written from seed 0), a 32-slot MultiLLM at context 2304 with an
1800-token prompt in slot 0.  Timed with a host clock around each call (every call ends in a device synchronise; best of --reps
after one warm-up): the prompt's eval, MultiLLM.fork of slot 0 into the other 31 slots, MultiLLM.save of slot 0 and
MultiLLM.restore into slot 1 (each with the bytes moved), and generate_many of 8 samples of 64 new tokens of the prompt, with
n = 8 (one prompt eval, then forks) against 8 copies of the prompt.  Also printed: the GPU, its power limit and maximum SM clock.
Asserts that the restored and forked slots pick the same greedy tokens as slot 0."""
import argparse
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import Config, MultiLLM, synth  # noqa: E402

CTX, PROMPT, SLOTS = 2304, 1800, 32


def best_of(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return 1e3 * min(times), 1e3 * float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.dir or tmp) / "llama7b_q4_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q4_K_M", seed=0)
        prompt = np.random.default_rng(100).integers(259, synth.LLAMA2_7B.n_vocab, PROMPT).tolist()
        prompt[0] = 1
        m = MultiLLM(str(path), n_slots=SLOTS, config=Config(context_length=CTX))

        def eval_prompt():
            m.reset(0)
            m.eval({0: prompt}, batch_size=512)
        ms, med = best_of(eval_prompt, a.reps)
        print(f"eval of the {PROMPT}-token prompt into one slot: {ms:.1f} ms (median {med:.1f})", flush=True)

        dsts = list(range(1, SLOTS))
        ms, med = best_of(lambda: m.fork(0, dsts), a.reps)
        print(f"fork 1 -> {len(dsts)} slots (each slot's whole K / V region): {ms:.1f} ms (median {med:.1f})", flush=True)

        st = m.save(0)
        ms, med = best_of(lambda: m.save(0), a.reps)
        print(f"save of one slot at n_past {PROMPT}: {ms:.1f} ms (median {med:.1f}), {len(st.data) / 1e6:.0f} MB "
              f"({len(st.data) / ms / 1e6:.1f} GB/s)", flush=True)
        ms, med = best_of(lambda: m.restore(1, st), a.reps)
        print(f"restore of that state into another slot: {ms:.1f} ms (median {med:.1f}) ({len(st.data) / ms / 1e6:.1f} GB/s)", flush=True)

        picks = []
        for _ in range(4):
            picks.append(m.greedy([0, 1, 5]))
            m.eval({s: [p] for s, p in zip((0, 1, 5), picks[-1])})
        assert all(p[0] == p[1] == p[2] for p in picks), picks

        kw = dict(top_k=40, top_p=0.95, temperature=0.8, repetition_penalty=1.1, batch_size=512)
        seeds = list(range(8))
        ms_f, _ = best_of(lambda: m.generate_many([prompt], 64, n=8, seeds=seeds, **kw), max(1, a.reps // 2))
        ms_c, _ = best_of(lambda: m.generate_many([prompt] * 8, 64, seed=0, **kw), max(1, a.reps // 2))
        print(f"generate_many, 8 samples x 64 new tokens of the prompt: n=8 with forks {ms_f:.0f} ms, 8 copies of the prompt "
              f"{ms_c:.0f} ms ({ms_c / ms_f:.2f}x)", flush=True)
        del m
        if not a.dir:
            path.unlink()


if __name__ == "__main__":
    main()
