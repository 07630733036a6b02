"""Writes what the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built by oracle/Makefile where the reference
sources are available) computes on the head_dims_refs model cases:  python tests/golden/make_golden_head_dims.py

  head_dims_runs.npz  per case and batch size: greedy tokens and SHA-256 digests of the logits and embeddings after the prompt
                      and of the last logits

The files of the other generators are not touched.
"""
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import head_dims_refs as H  # noqa: E402
import modelcases  # noqa: E402
import refs  # noqa: E402


def runs(tmp):
    from ctransformers_b200 import AutoModelForCausalLM
    out = {}
    for name, case in H.all_cases().items():
        path, ctx = H.build_model(name, tmp)
        for bs in case[5]:
            llm = AutoModelForCausalLM.from_pretrained(str(path), lib=str(refs.REF_SO), context_length=ctx, threads=8)
            first_logits, first_embd, toks, last_logits, gaps = modelcases.run_greedy(llm, H.prompt_for(name), H.N_NEW, batch_size=bs)
            for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
                out[f"{name}_bs{bs}_{k}"] = np.array(refs.digest(v))
            out[f"{name}_bs{bs}_tokens"] = np.array(toks, np.int32)
            print(name, bs, "tokens", toks, "min top-2 gap", min(gaps), flush=True)
    np.savez_compressed(HERE / "head_dims_runs.npz", **out)


if __name__ == "__main__":
    assert refs.have_ref(), "build oracle/_ref first: make -C oracle ref"
    with tempfile.TemporaryDirectory() as tmp:
        runs(tmp)
    print("golden runs written to", HERE)
