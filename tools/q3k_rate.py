#!/usr/bin/env python
"""Device-timed rates of a 7B-shaped Llama file in Q3_K_M (synth.LLAMA2_7B, random valid blocks, as the reference's quantizer
assigns the types): python tools/q3k_rate.py [--dir DIR] [--steps N]

Prints the GPU, its power limit and maximum SM clock, then the greedy decode rate (ctb_llm_decode_greedy, median of 5), the rate
of a 2048-token prompt through llm.eval(tokens, batch_size=512) at context 2304 (ctb_llm_last_eval_ms, median of 5) and the
weight bytes a decoded token streams.  The file (3.3 GB) is written to --dir (default: a temporary directory, removed afterwards)."""
import argparse
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import AutoModelForCausalLM, synth  # noqa: E402

PROMPT = [1] + list(range(300, 331))


def decode_rate(path, steps):
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=512)
    llm.eval(PROMPT, batch_size=8)
    first = llm.sample(top_k=1, repetition_penalty=1.0, seed=0)
    out = (C.c_int * max(steps, 16))()
    llm.ctb_llm_decode_greedy(first, len(PROMPT), 16, out)                          # warm-up
    ms = sorted(llm.ctb_llm_decode_greedy(first, len(PROMPT), steps, out) for _ in range(5))
    return steps / (ms[2] / 1e3), ms[2] / steps, llm.ctb_llm_weight_bytes_per_token()


def prompt_rate(path, n_prompt=2048, ctx=2304):
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    ids = np.random.default_rng(1).integers(259, synth.LLAMA2_7B.n_vocab, n_prompt).tolist()
    ids[0] = 1

    def once():
        llm._context = []
        llm.eval(ids, batch_size=512)
        return llm.ctb_llm_last_eval_ms()
    once()                                                                          # warm-up
    ms = sorted(once() for _ in range(5))
    return n_prompt / (ms[2] / 1e3), ms[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--steps", type=int, default=128)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.dir or tmp) / "llama7b_q3_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q3_K_M", seed=1)
        tps, ms, wb = decode_rate(path, a.steps)
        print(f"Q3_K_M decode: {tps:.1f} tokens/s  step {ms:.3f} ms  weight_bytes_per_token {wb / 1e9:.3f} GB  {wb / ms / 1e6:.0f} GB/s", flush=True)
        ptps, pms = prompt_rate(path)
        print(f"Q3_K_M 2048-token prompt: {ptps:.0f} tokens/s  ({pms:.1f} ms)", flush=True)
        path.unlink()


if __name__ == "__main__":
    main()
