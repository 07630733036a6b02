"""Regenerates tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built from the
reference sources by oracle/Makefile).  Run where those sources are available:  python tests/golden/make_golden.py

Contents
  kat_quant.npz    seeded activations → the reference's Q8_K / Q8_0 block bytes; seeded weights quantized by the
                   reference → its vec_dot result per type (known-answer vectors for oracle and CUDA kernels)
  model_<case>.npz prompt, last-token logits / embeddings after the prompt, 24 greedy tokens, final logits, top-2 gaps
                   for each synthetic model in tests/modelcases.py (weights come from seeded random blocks, so the GGUF
                   is reproducible without the reference)
  host_logic.npz   tokenizer ids for a set of strings, detokenized pieces, and sampler picks for seeded logits
  reference_blocks.npz  blocks written by the reference's quantizer, the pool of refs.reference_quantized_blocks
  reference_runs.npz  what the reference computed for each test that compares with it (tests/test_model_gpu.py,
                   tests/test_oracle.py, tests/test_long_context_gpu.py), so those tests run where the reference is not
                   available.  `python make_golden.py long_context` adds the long-context runs to the existing file,
                   `python make_golden.py realq_prefill` the reference-quantized Q5_K_M prefill runs, `python make_golden.py
                   norm_order` the runs of the models with planted norm rows (tests/test_norm_order_gpu.py).
"""
import ctypes as C
import json
import os
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import modelcases  # noqa: E402
import refs  # noqa: E402
from refs import Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0, Q8_K, ptr  # noqa: E402

TEXTS = ["AI is going to", "  hello  world ", "héllo ☃ the", "", "theof and123", "a\nb\tc", "The people of the water were very little.",
         "that's what they'll've said", "12345 67", "\x00\x01"]


def kat_quant():
    rng = np.random.default_rng(2024)
    out = {}
    for k in (256, 1024):
        x = (rng.standard_normal(k) * 3).astype(np.float32)
        out[f"x_{k}"] = x
        out[f"q8k_{k}"] = refs.ref_quantize_act(Q8_K, x)
        out[f"q80_{k}"] = refs.ref_quantize_act(Q8_0, x)
    k, m = 1024, 6
    w = (rng.standard_normal((m, k)) * 0.05).astype(np.float32)
    x = out["x_1024"]
    out["w_f32"] = w
    for t, at in ((Q4_0, Q8_0), (Q8_0, Q8_0), (Q4_K, Q8_K), (Q5_K, Q8_K), (Q6_K, Q8_K), (Q5_0, Q8_0)):   # (appended: earlier vectors keep their bytes)
        wq = refs.ref_quantize(t, w).reshape(m, -1)
        act = refs.ref_quantize_act(at, x)
        out[f"wq_{t}"] = wq
        out[f"dot_{t}"] = np.array([refs.ref_vec_dot(t, k, wq[i], act) for i in range(m)], np.float32)
        deq = np.zeros((m, k), np.float32)
        refs.ref_traits(t)["to_float"](ptr(wq), ptr(deq), m * k)
        out[f"deq_{t}"] = deq
    np.savez_compressed(HERE / "kat_quant.npz", **out)


def ref_llm(path, ctx, threads=4):
    from ctransformers_b200 import AutoModelForCausalLM
    return AutoModelForCausalLM.from_pretrained(str(path), lib=str(refs.REF_SO), context_length=ctx, threads=threads)


def models(tmp, only=None):
    for name in modelcases.CASES:
        if only and name not in only:
            continue
        path, ctx = modelcases.build(name, tmp)
        llm = ref_llm(path, ctx)
        prompt = modelcases.prompt_for(name)
        first_logits, first_embd, toks, last_logits, gaps = modelcases.run_greedy(llm, prompt, modelcases.N_NEW)
        np.savez_compressed(HERE / f"model_{name}.npz", prompt=np.array(prompt), first_logits=first_logits, first_embd=first_embd,
                            tokens=np.array(toks), last_logits=last_logits, gaps=np.array(gaps))
        print(name, "tokens", toks[:8], "min top-2 gap", min(gaps))


def host_logic(tmp):
    out = {}
    for name in ("llama_tiny_q4km", "falcon_tiny_q5km"):
        path, ctx = modelcases.build(name, tmp)
        llm = ref_llm(path, ctx)
        for i, text in enumerate(TEXTS):
            if name.startswith("falcon") and not text.isascii():
                continue   # the synthetic BPE vocabulary only holds printable ASCII bytes
            if name.startswith("falcon") and any(ord(c) < 33 and c not in " " for c in text):
                continue
            ids = llm.tokenize(text)
            out[f"{name}_tok_{i}"] = np.array(ids, np.int32)
        pieces = [llm.detokenize([t], decode=False) for t in range(llm.vocab_size)]
        out[f"{name}_pieces"] = np.array([p.hex() for p in pieces])
        # sampler: seeded logits written through the mutable logits view, then sampled with several settings
        llm.eval([5, 6, 7])
        rng = np.random.default_rng(3)
        picks = []
        settings = [(40, 0.95, 0.8, 1.1, 1), (1, 1.0, 1.0, 1.0, 0), (5, 0.5, 1.3, 1.3, 7), (0, 0.9, 0.7, 1.0, 123), (1000, 1.0, 0.01, 1.2, 9)]
        lg_all = []
        for rep in range(4):
            lg = (rng.standard_normal(llm.vocab_size) * 3).astype(np.float32)
            lg_all.append(lg)
            view = llm.logits
            for j, v in enumerate(lg):
                view[j] = float(v)
            for (k, p, temp, pen, seed) in settings:
                picks.append(llm.sample(top_k=k, top_p=p, temperature=temp, repetition_penalty=pen, last_n_tokens=64, seed=seed))
        out[f"{name}_sample_logits"] = np.array(lg_all)
        out[f"{name}_sample_picks"] = np.array(picks, np.int32)
        out[f"{name}_sample_settings"] = np.array(settings, np.float64)
    out["texts"] = np.array(TEXTS)
    np.savez_compressed(HERE / "host_logic.npz", **out)


def reference_blocks():
    """Blocks the reference's quantizer wrote (refs.reference_quantized_blocks draws matrices from them): 256 K-quant blocks
    and 1024 32-weight blocks per type, quantized from seeded rows whose scale spans 0.005 .. 2 and whose mean is offset, so
    the scale / min / sign bit patterns of the quantizers all occur."""
    out = {}
    for t in (Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K):
        rows = 64 if t in (Q4_K, Q5_K, Q6_K) else 32
        rng = np.random.default_rng(100 + t)
        scale = np.exp(rng.uniform(np.log(0.005), np.log(2.0), (rows, 1)))
        w = (rng.standard_normal((rows, 1024)) * scale + rng.uniform(-0.5, 0.5, (rows, 1)) * scale).astype(np.float32)
        bs, sz = refs.BLOCK[t]
        out[f"blocks_{t}"] = refs.ref_quantize(t, w).reshape(-1, sz)
    np.savez_compressed(HERE / "reference_blocks.npz", **out)


def reference_runs(tmp):
    """The reference's results for the tests that compare with it, keyed by test.  Float vectors and quantized blocks are
    stored as SHA-256 digests of their bytes (refs.digest): the comparison stays bit-exact at 64 bytes per vector."""
    out = {}

    def greedy(key, run):
        first_logits, first_embd, toks, last_logits, _ = run
        for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
            out[f"{key}_{k}"] = np.array(refs.digest(v))
        out[f"{key}_tokens"] = np.array(toks, np.int32)

    # tests/test_model_gpu.py
    for name in ("llama_tiny_q4km", "llama_gqa_q5km", "falcon_tiny_q5km"):
        path, ctx = modelcases.build(name, tmp)
        for bs in (8, 64, 5):
            greedy(f"live_{name}_bs{bs}", modelcases.run_greedy(ref_llm(path, ctx), modelcases.prompt_for(name), modelcases.N_NEW, batch_size=bs))
    for name, bs in (("llama_wide_q4km", 512), ("llama_wide_q4km", 64), ("llama_gqa_q5km", 5), ("falcon_tiny_q5km", 512)):
        path, _ = modelcases.build(name, tmp)
        greedy(f"prefill_{name}_bs{bs}", modelcases.run_greedy(ref_llm(path, 96), modelcases.long_prompt(name), 6, batch_size=bs))
    greedy("realq", modelcases.run_greedy(ref_llm(modelcases.build_realq(tmp), 64), modelcases.REALQ_PROMPT, 8))
    import bench
    for workload in ("llama2-7b", "falcon7b"):
        bench.WL = bench.WORKLOADS[workload]
        path = bench.ensure_model(0, 1, lambda: None)
        llm = ref_llm(path, 128, threads=min(16, os.cpu_count() or 1))
        greedy(f"bench_{workload}", modelcases.run_greedy(llm, bench.prompt_ids()[:32], 8))
        del llm
    # tests/test_oracle.py
    for name in ("llama_tiny_q4km", "falcon_tiny_q5km"):
        path, ctx = modelcases.build(name, tmp)
        ids = modelcases.long_prompt(name, bos=False)
        for bs in (8, 64, 33):
            llm = ref_llm(path, ctx)
            llm.eval(ids, batch_size=bs)
            steps = []
            for _ in range(3):
                steps.append(np.array(llm.logits, dtype=np.float32))
                llm.eval([int(np.argmax(steps[-1]))])
            out[f"chunked_{name}_bs{bs}_logits"] = np.array([refs.digest(s) for s in steps])
    rng = np.random.default_rng(7)
    q8k, q80 = [], []
    for trial in range(60):
        x = (rng.standard_normal(2048) * rng.choice([1e-3, 1, 50])).astype(np.float32)
        if trial % 7 == 0:
            x[256:512] = 0
        q8k.append(refs.digest(refs.ref_quantize_act(Q8_K, x)))
        q80.append(refs.digest(refs.ref_quantize_act(Q8_0, x)))
    out["act_quant_q8_K"], out["act_quant_q8_0"] = np.array(q8k), np.array(q80)
    for t, at in ((Q4_0, Q8_0), (Q5_0, Q8_0), (Q8_0, Q8_0), (Q4_K, Q8_K), (Q5_K, Q8_K), (Q6_K, Q8_K)):
        k = 4096
        wq = refs.reference_quantized_blocks(t, k, 16, seed=t).reshape(16, -1)
        act = refs.ref_quantize_act(at, np.random.default_rng(t).standard_normal(k).astype(np.float32))
        out[f"vec_dot_{t}"] = np.array([refs.ref_vec_dot(t, k, wq[i], act) for i in range(16)], np.float32)
        from ctransformers_b200 import synth
        blocks = np.ascontiguousarray(synth.random_blocks(t, 1024, 8, 0.02, np.random.default_rng(t)))
        deq = np.zeros(8 * 1024, np.float32)
        refs.ref_traits(t)["to_float"](ptr(blocks), ptr(deq), deq.size)
        out[f"random_blocks_{t}_dequant"] = np.array(refs.digest(deq))
    np.savez_compressed(HERE / "reference_runs.npz", **out)


def long_context_runs(tmp):
    """Adds the reference's results for modelcases.LONG_RUNS to reference_runs.npz as keys long_<run>_*; every key already in
    the file keeps its bytes (the rest of reference_runs() also rebuilds the 7B-shaped bench models)."""
    old = dict(refs.golden_runs())
    out = dict(old)

    for key, (name, ctx, n_prompt, bs, n_new) in modelcases.LONG_RUNS.items():
        path, _ = modelcases.build(name, tmp)
        run = modelcases.run_greedy(ref_llm(path, ctx, threads=min(16, os.cpu_count() or 1)), modelcases.seeded_prompt(name, n_prompt), n_new,
                                    batch_size=bs)
        first_logits, first_embd, toks, last_logits, _ = run
        for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
            out[f"long_{key}_{k}"] = np.array(refs.digest(v))
        out[f"long_{key}_tokens"] = np.array(toks, np.int32)
        print(key, "tokens", toks[:8])
    np.savez_compressed(HERE / "reference_runs.npz", **out)
    new = refs.golden_runs()
    assert all(np.array_equal(new[k], v) and new[k].dtype == v.dtype for k, v in old.items()), "an existing key changed"


def realq_prefill_runs(tmp):
    """Adds the reference's results for modelcases.REALQ_PREFILL to reference_runs.npz as keys prefill_<key>_*; every key already
    in the file keeps its bytes."""
    old = dict(refs.golden_runs())
    out = dict(old)
    for key, (arch, ftype) in modelcases.REALQ_PREFILL.items():
        path = modelcases.build_realq(tmp, arch, ftype)
        run = modelcases.run_greedy(ref_llm(path, modelcases.REALQ_PREFILL_CTX), modelcases.realq_prompt(arch), modelcases.REALQ_PREFILL_NEW,
                                    batch_size=512)
        first_logits, first_embd, toks, last_logits, _ = run
        for k, v in (("first_logits", first_logits), ("first_embd", first_embd), ("last_logits", last_logits)):
            out[f"prefill_{key}_{k}"] = np.array(refs.digest(v))
        out[f"prefill_{key}_tokens"] = np.array(toks, np.int32)
        print(key, "tokens", toks)
    np.savez_compressed(HERE / "reference_runs.npz", **out)
    new = refs.golden_runs()
    assert all(np.array_equal(new[k], v) and new[k].dtype == v.dtype for k, v in old.items()), "an existing key changed"


def norm_order_runs(tmp):
    """Adds the reference's results for modelcases.NORM_ORDER_MODELS to reference_runs.npz as keys norm_<case>_*; every key
    already in the file keeps its bytes."""
    old = dict(refs.golden_runs())
    out = dict(old)
    for name in modelcases.NORM_ORDER_MODELS:
        path, ctx = modelcases.build_norm_order(name, tmp)
        states, toks = modelcases.norm_order_llm_run(ref_llm(path, ctx), name)
        for i, (logits, embd) in enumerate(states):
            out[f"norm_{name}_{i}_logits"] = np.array(refs.digest(logits))
            out[f"norm_{name}_{i}_embd"] = np.array(refs.digest(embd))
        out[f"norm_{name}_tokens"] = np.array(toks, np.int32)
        print(name, "tokens", toks)
    np.savez_compressed(HERE / "reference_runs.npz", **out)
    new = refs.golden_runs()
    assert all(np.array_equal(new[k], v) and new[k].dtype == v.dtype for k, v in old.items()), "an existing key changed"


if __name__ == "__main__":
    assert refs.have_ref(), "build oracle/_ref first: make -C oracle ref"
    import sys
    only = sys.argv[1:]          # python make_golden.py [model case ...]: regenerate only those model fixtures
    with tempfile.TemporaryDirectory() as tmp:
        if only:                 # "kat" regenerates kat_quant.npz (its vectors are appended per type, earlier ones keep their bytes)
            if "kat" in only:
                kat_quant()
            if "reference_blocks" in only:
                reference_blocks()
            if "reference_runs" in only:
                reference_runs(tmp)
            if "long_context" in only:
                long_context_runs(tmp)
            if "realq_prefill" in only:
                realq_prefill_runs(tmp)
            if "norm_order" in only:
                norm_order_runs(tmp)
            cases = [o for o in only if o not in ("kat", "reference_blocks", "reference_runs", "long_context", "realq_prefill", "norm_order")]
            if cases:
                models(tmp, cases)
        else:
            kat_quant()
            models(tmp)
            host_logic(tmp)
            reference_blocks()
            reference_runs(tmp)
    print("golden vectors written to", HERE)
