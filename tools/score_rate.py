#!/usr/bin/env python
"""What scoring costs: python tools/score_rate.py [--dir DIR] [--reps N]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, seed 0) and the Falcon-7B-shaped Q5_K_M file (synth.FALCON_7B_SHAPED,
seed 0), at context 2304:
  * LLM.score of a 2048-token sequence at batch_size 512 (every token's row reduced on the device), in tokens/s;
  * the only way without rows: one eval per token, each followed by a read of the last logits (timed over the first 256 tokens);
  * MultiLLM.score_many of 32 requests of a 200-token context and a 20-token continuation on a 32-slot handle.
Host clock around each call (every call ends in a device synchronise); best of --reps after one warm-up.  Also printed: the GPU,
its power limit and maximum SM clock."""
import argparse
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import AutoModelForCausalLM, Config, MultiLLM, synth  # noqa: E402

CTX, N_SCORE, N_SINGLE, N_REQ, REQ_CTX, REQ_CONT = 2304, 2048, 256, 32, 200, 20


def best_of(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times), float(np.median(times))


def measure(path, arch, n_vocab, reps):
    lo = 259 if arch == "llama" else 0
    rng = np.random.default_rng(100)
    toks = rng.integers(lo, n_vocab, N_SCORE).tolist()
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=CTX)

    def score():
        llm._context = []
        llm.score(toks, batch_size=512)
    s, med = best_of(score, reps)
    print(f"  LLM.score, {N_SCORE} tokens: {s * 1e3:.0f} ms (median {med * 1e3:.0f}), {N_SCORE / s:.0f} tokens/s", flush=True)

    def one_by_one():
        llm._context = []
        for t in toks[:N_SINGLE]:
            llm.eval([t])
            llm.ctransformers_llm_logits_data()[0]
    s1, med1 = best_of(one_by_one, max(1, reps // 2))
    print(f"  one eval per token ({N_SINGLE} tokens): {s1 * 1e3 / N_SINGLE:.2f} ms per token (median {med1 * 1e3 / N_SINGLE:.2f}), "
          f"{N_SINGLE / s1:.0f} tokens/s; LLM.score is {(N_SCORE / s) / (N_SINGLE / s1):.1f}x", flush=True)
    del llm

    m = MultiLLM(str(path), n_slots=N_REQ, config=Config(context_length=512))
    reqs = [(rng.integers(lo, n_vocab, REQ_CTX).tolist(), rng.integers(lo, n_vocab, REQ_CONT).tolist()) for _ in range(N_REQ)]
    s2, med2 = best_of(lambda: m.score_many(reqs, batch_size=512), reps)
    n_tok = N_REQ * (REQ_CTX + REQ_CONT - 1)
    print(f"  MultiLLM.score_many, {N_REQ} requests of {REQ_CTX} + {REQ_CONT} tokens: {s2 * 1e3:.0f} ms (median {med2 * 1e3:.0f}), "
          f"{n_tok / s2:.0f} tokens/s", flush=True)
    del m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        d = Path(a.dir or tmp)
        for arch, shape, ftype, name in (("llama", synth.LLAMA2_7B, "Q4_K_M", "llama7b_q4_k_m.gguf"),
                                         ("falcon", synth.FALCON_7B_SHAPED, "Q5_K_M", "falcon7b_q5_k_m.gguf")):
            path = d / name
            if not path.exists():
                (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=0)
            print(f"{name}:", flush=True)
            measure(path, arch, shape.n_vocab, a.reps)
            if not a.dir:
                path.unlink()


if __name__ == "__main__":
    main()
