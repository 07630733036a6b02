#!/usr/bin/env python
"""Device-timed greedy decode rate of 7B-shaped Llama files in Q4_0, Q4_1 and Q5_1 (all matrices in the type, Q6_K head, random
valid blocks): python tools/q1_decode_rate.py [--dir DIR] [--steps N]

All three run on k_matvec, whose HBM traffic is the weight planes: Q4_1 carries 20 bytes per 32 weights against Q4_0's 18 and
Q5_1 24, so a bandwidth-bound Q4_1 decode runs at about 18/20 of Q4_0's rate.  Prints the GPU, its power limit and one line per
file.  The files (4 to 5 GB each) are written to --dir (default: a temporary directory, removed afterwards)."""
import argparse
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import AutoModelForCausalLM, synth  # noqa: E402

PROMPT = [1] + list(range(300, 331))


def rate(path, steps):
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=512)
    llm.eval(PROMPT, batch_size=8)
    first = llm.sample(top_k=1, repetition_penalty=1.0, seed=0)
    out = (C.c_int * max(steps, 16))()
    llm.ctb_llm_decode_greedy(first, len(PROMPT), 16, out)                          # warm-up
    ms = sorted(llm.ctb_llm_decode_greedy(first, len(PROMPT), steps, out) for _ in range(5))
    return steps / (ms[2] / 1e3), ms[2] / steps, llm.ctb_llm_weight_bytes_per_token()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--steps", type=int, default=128)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        d = Path(a.dir or tmp)
        res = {}
        for ftype in ("Q4_0", "Q4_1", "Q5_1"):
            path = d / f"llama7b_{ftype.lower()}.gguf"
            if not path.exists():
                synth.write_llama(path, synth.LLAMA2_7B, ftype, seed=1)
            res[ftype] = rate(path, a.steps)
            tps, ms, wb = res[ftype]
            print(f"{ftype}: {tps:.1f} tokens/s  step {ms:.3f} ms  weights {wb / 1e9:.3f} GB/token  {wb / ms / 1e6:.0f} GB/s", flush=True)
            path.unlink()
        print(f"Q4_1 / Q4_0 rate {res['Q4_1'][0] / res['Q4_0'][0]:.3f} (byte ratio 18/20 = 0.900); "
              f"Q5_1 / Q4_0 {res['Q5_1'][0] / res['Q4_0'][0]:.3f} (18/24 = 0.750)")


if __name__ == "__main__":
    main()
