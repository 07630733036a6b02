#!/usr/bin/env python
"""Aggregate decode rate of many sequences on one GPU (MultiLLM, batched launches) against the single-sequence step kernel:
python tools/multi_rate.py [--dir DIR] [--steps N] [--slots 1,2,4,8,16,32]

On the 7B-shaped Q4_K_M file bench.py decodes (synth.LLAMA2_7B, written from seed 0): for each slot count S, S prompts are
evaluated together, then after a warm-up, N lockstep greedy steps (ctb_multi_eval of one token per slot + ctb_multi_greedy) are
timed with CUDA events (ctb_multi_last_eval_ms per step, summed).  Line 1: context 512, 256-token prompts.  Line 2: context 2304,
1800-token prompts, where attention over ~1900 positions per token dominates.  Also printed: the GPU, its power limit and
maximum SM clock, and in the same process the single-sequence ctb_llm_decode_greedy rate.  Asserts that the greedy tokens of a
few slots equal the single-sequence run of the same prompt."""
import argparse
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from ctransformers_b200 import AutoModelForCausalLM, Config, MultiLLM, synth  # noqa: E402

WARMUP = 4


def prompts(n_slots, n_prompt):
    out = []
    for s in range(n_slots):
        ids = np.random.default_rng(100 + s).integers(259, synth.LLAMA2_7B.n_vocab, n_prompt).tolist()
        ids[0] = 1
        out.append(ids)
    return out


def single_rate(path, ctx, prompt, steps):
    """ctb_llm_decode_greedy after the same prompt: tokens/s, ms per step, and the greedy tokens."""
    llm = AutoModelForCausalLM.from_pretrained(str(path), context_length=ctx)
    llm.eval(prompt, batch_size=512)
    first = llm.sample(top_k=1, repetition_penalty=1.0, seed=0)
    out = (C.c_int * max(steps, 16))()
    llm.ctb_llm_decode_greedy(first, len(prompt), 16, out)                      # warm-up
    ms = llm.ctb_llm_decode_greedy(first, len(prompt), steps, out)
    toks = [first] + list(out[: steps - 1])
    del llm
    return steps / (ms / 1e3), ms / steps, toks


def multi_rate(m, ps, steps):
    """S prompts together, WARMUP lockstep steps, then `steps` timed ones.  Returns tokens/s, ms per step, greedy tokens per slot."""
    S = len(ps)
    for s in range(S):
        m.reset(s)
    m.eval(dict(enumerate(ps)), batch_size=512)
    toks = [[] for _ in range(S)]
    ms = 0.0
    for i in range(WARMUP + steps):
        picks = m.greedy(range(S))
        for s, t in enumerate(picks):
            toks[s].append(t)
        launches = m.launches()
        m.eval({s: [t] for s, t in enumerate(picks)})
        assert m.launches() == launches + -(-S // 32)
        if i >= WARMUP:
            ms += m.last_eval_ms()
    return S * steps / (ms / 1e3), ms / steps, toks


def line(path, ctx, n_prompt, steps, slots):
    ps = prompts(max(slots), n_prompt)
    tps1, ms1, ref_toks = single_rate(path, ctx, ps[0], WARMUP + steps)
    print(f"ctx {ctx}, prompt {n_prompt}: single-sequence ctb_llm_decode_greedy {tps1:.1f} tokens/s ({ms1:.3f} ms/step)", flush=True)
    m = MultiLLM(str(path), n_slots=max(slots), config=Config(context_length=ctx))
    for S in slots:
        tps, ms, toks = multi_rate(m, ps[:S], steps)
        assert toks[0] == ref_toks, f"S={S}: slot 0's greedy tokens differ from the single-sequence run"
        print(f"ctx {ctx}, prompt {n_prompt}: S={S:2d}  {tps:8.1f} tokens/s aggregate  {ms:7.3f} ms/step  ({tps / tps1:.2f}x single)", flush=True)
    if max(slots) > 1:                                     # a second slot against its own single-sequence run
        s = min(3, max(slots) - 1)
        _, _, want = single_rate(path, ctx, ps[s], WARMUP + steps)
        assert toks[s] == want, f"slot {s}: greedy tokens differ from the single-sequence run"
    del m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--slots", default="1,2,4,8,16,32")
    ap.add_argument("--long-slots", default="1,8,32")
    a = ap.parse_args()
    slots = [int(x) for x in a.slots.split(",")]
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(a.dir or tmp) / "llama7b_q4_k_m.gguf"
        if not path.exists():
            synth.write_llama(path, synth.LLAMA2_7B, "Q4_K_M", seed=0)
        line(path, 512, 256, a.steps, slots)
        if a.long_slots:
            line(path, 2304, 1800, a.steps, [int(x) for x in a.long_slots.split(",")])
        if not a.dir:
            path.unlink()


if __name__ == "__main__":
    main()
