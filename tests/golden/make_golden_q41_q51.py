"""Writes the Q4_1 / Q5_1 golden vectors from the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built by
oracle/Makefile where the reference sources are available):  python tests/golden/make_golden_q41_q51.py

  kat_q8_1.npz        planted activation rows (q41_q51_refs.planted_rows) -> the reference's Q8_1 block bytes; seeded weights
                      quantized to Q4_1 / Q5_1 by the reference, reference-quantized and edge blocks, each row's vec_dot with the
                      Q8_1 image of seeded activations, and the reference's dequantized rows
  q41_q51_blocks.npz  1024 blocks per type written by the reference's quantizer from rows of scale 0.002 .. 0.1 with offset means
                      (q41_q51_refs.reference_quantized_blocks)
  q41_q51_runs.npz    what the reference computed on every q41_q51_refs model case at batch sizes 8 / 64 / 5: greedy tokens and
                      SHA-256 digests of the logits and embeddings after the prompt and of the last logits

The files of make_golden.py are not touched.
"""
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import q41_q51_refs as Q  # noqa: E402
import refs  # noqa: E402
from refs import ptr  # noqa: E402

KAT_K, KAT_M = 1024, 8


def kat():
    out = {}
    for k in (32, 1024, 4544):
        rows = Q.planted_rows(k, seed=k)
        out[f"x_{k}"] = rows
        out[f"q81_{k}"] = np.stack([refs.ref_quantize_act(Q.Q8_1, x) for x in rows])
    rng = np.random.default_rng(31)
    x = (rng.standard_normal((3, KAT_K)) * np.array([[0.01], [1.0], [30.0]])).astype(np.float32)
    out["dot_x"] = x
    acts = [refs.ref_quantize_act(Q.Q8_1, r) for r in x]
    w = (rng.standard_normal((KAT_M, KAT_K)) * 0.05 + rng.uniform(-0.05, 0.05, (KAT_M, 1))).astype(np.float32)
    for t in (Q.Q4_1, Q.Q5_1):
        for src, wq in (("refq", refs.ref_quantize(t, w)), ("pool", Q.reference_quantized_blocks(t, KAT_K, KAT_M, seed=t)),
                        ("edge", Q.edge_blocks(t, KAT_K, KAT_M, seed=t))):
            wq = wq.reshape(KAT_M, -1)
            out[f"w_{src}_{t}"] = wq
            out[f"dot_{src}_{t}"] = np.array([[refs.ref_vec_dot(t, KAT_K, wq[i], a) for i in range(KAT_M)] for a in acts], np.float32)
            deq = np.zeros((KAT_M, KAT_K), np.float32)
            refs.ref_traits(t)["to_float"](ptr(np.ascontiguousarray(wq)), ptr(deq), deq.size)
            out[f"deq_{src}_{t}"] = deq
    np.savez_compressed(HERE / "kat_q8_1.npz", **out)


def blocks():
    out = {}
    for t in (Q.Q4_1, Q.Q5_1):
        rng = np.random.default_rng(200 + t)
        scale = np.exp(rng.uniform(np.log(0.002), np.log(0.1), (32, 1)))   # weights of a model that stays finite and untied
        w = (rng.standard_normal((32, 1024)) * scale + rng.uniform(-0.5, 0.5, (32, 1)) * scale).astype(np.float32)
        out[f"blocks_{t}"] = refs.ref_quantize(t, w).reshape(-1, refs.BLOCK[t][1])
    np.savez_compressed(HERE / "q41_q51_blocks.npz", **out)


def runs(tmp):
    import modelcases
    from ctransformers_b200 import AutoModelForCausalLM
    out = {}
    for name in Q.model_cases():
        path, ctx = Q.build_model(name, tmp)
        for bs in Q.BATCH_SIZES:
            llm = AutoModelForCausalLM.from_pretrained(str(path), lib=str(refs.REF_SO), context_length=ctx, threads=4)
            first_logits, first_embd, toks, last_logits, gaps = modelcases.run_greedy(llm, Q.prompt_for(name), Q.N_NEW, batch_size=bs)
            for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
                out[f"{name}_bs{bs}_{k}"] = np.array(refs.digest(v))
            out[f"{name}_bs{bs}_tokens"] = np.array(toks, np.int32)
            print(name, bs, "tokens", toks[:8], "min top-2 gap", min(gaps))
    np.savez_compressed(HERE / "q41_q51_runs.npz", **out)


if __name__ == "__main__":
    assert refs.have_ref(), "build oracle/_ref first: make -C oracle ref"
    blocks()
    kat()
    with tempfile.TemporaryDirectory() as tmp:
        runs(tmp)
    print("golden vectors written to", HERE)
