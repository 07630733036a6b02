"""Writes the Q3_K golden vectors from the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built by oracle/Makefile
where the reference sources are available):  python tests/golden/make_golden_q3k.py

  q3k_blocks.npz  512 Q3_K blocks written by the reference's quantizer from rows of scale 0.002 .. 0.1 with offset means
                  (q3k_refs.reference_quantized_blocks)
  q3k_kat.npz     seeded activation rows and their Q8_K bytes from the reference; for random, reference-quantized and edge blocks
                  (q3k_refs.blocks) each row's vec_dot with those activations, and the reference's dequantized rows
  q3k_runs.npz    what the reference computed on every q3k_refs model case and batch size: greedy tokens and SHA-256 digests of
                  the logits and embeddings after the prompt and of the last logits

The files of the other generators are not touched.
"""
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import modelcases  # noqa: E402
import q3k_refs as Q  # noqa: E402
import refs  # noqa: E402
from refs import ptr  # noqa: E402

KAT_K, KAT_M = 2048, 16


def blocks():
    rng = np.random.default_rng(311)
    scale = np.exp(rng.uniform(np.log(0.002), np.log(0.1), (32, 1)))
    w = (rng.standard_normal((32, 4096)) * scale + rng.uniform(-0.5, 0.5, (32, 1)) * scale).astype(np.float32)
    np.savez_compressed(HERE / "q3k_blocks.npz", blocks=refs.ref_quantize(Q.Q3_K, w).reshape(-1, 110))


def kat():
    out = {}
    rng = np.random.default_rng(37)
    x = (rng.standard_normal((4, KAT_K)) * np.array([[0.01], [1.0], [30.0], [1.0]])).astype(np.float32)
    x[3, 256:512] = 0                                            # an all-zero Q8_K block
    out["dot_x"] = x
    acts = np.stack([refs.ref_quantize_act(refs.Q8_K, r) for r in x])
    out["dot_q8k"] = acts
    for src in ("random", "refq", "edge"):
        wq = Q.blocks(src, KAT_K, KAT_M, seed=11).reshape(KAT_M, -1)
        out[f"w_{src}"] = wq
        out[f"dot_{src}"] = np.array([[refs.ref_vec_dot(Q.Q3_K, KAT_K, wq[i], a) for i in range(KAT_M)] for a in acts], np.float32)
        deq = np.zeros((KAT_M, KAT_K), np.float32)
        refs.ref_traits(Q.Q3_K)["to_float"](ptr(np.ascontiguousarray(wq)), ptr(deq), deq.size)
        out[f"deq_{src}"] = deq
    np.savez_compressed(HERE / "q3k_kat.npz", **out)


def runs(tmp):
    from ctransformers_b200 import AutoModelForCausalLM
    out = {}
    for name, case in Q.all_cases().items():
        path, ctx = Q.build_model(name, tmp)
        for bs in case[5]:
            llm = AutoModelForCausalLM.from_pretrained(str(path), lib=str(refs.REF_SO), context_length=ctx, threads=8)
            first_logits, first_embd, toks, last_logits, gaps = modelcases.run_greedy(llm, Q.prompt_for(name), Q.N_NEW, batch_size=bs)
            for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
                out[f"{name}_bs{bs}_{k}"] = np.array(refs.digest(v))
            out[f"{name}_bs{bs}_tokens"] = np.array(toks, np.int32)
            print(name, bs, "tokens", toks, "min top-2 gap", min(gaps), flush=True)
            del llm
        path.unlink()
    np.savez_compressed(HERE / "q3k_runs.npz", **out)


if __name__ == "__main__":
    assert refs.have_ref(), "build oracle/_ref first: make -C oracle ref"
    if "--runs-only" not in sys.argv:
        blocks()
        kat()
    with tempfile.TemporaryDirectory() as tmp:
        runs(tmp)
    print("golden vectors written to", HERE)
