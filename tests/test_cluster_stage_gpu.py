"""The decode-step kernel launched as clusters of two CTAs, which split every mat-vec input's norm and quantization between them
(csrc/matvec.cuh stage_q8k_pair), against the same kernel launched one CTA per cluster (CTB_ST_CLUSTER=0): the logits,
embeddings and greedy tokens of every step must be the same bits.  Each launch shape runs in a process of its own, because the
engine picks it once, when it loads a model.  The cases cover Q4_K_M and Q5_K_M weights, grouped-query attention, heads of
80 (the paired build for other head sizes), Falcon's LayerNorm, inputs with an odd number of Q8_K blocks (rank 0 then stages
one block more; at n_embd 256 rank 1 stages none), FFN widths 11008 and 18432 (the down input takes a second group of 16
elements per thread), a context past 512 (the step kernel's ring attention), and embedding rows whose fp64 norm sums round
differently in another order (refs.norm_order_rows), so that the exchanged partial sums and the element-order fallback both
run.  Programs with Q3_K matrices stay unpaired."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent

# name -> (builder, model case, prompt tokens, batch size, greedy steps, context); prompt None = the case's own prompt
RUNS = {
    "llama_tiny_q4km": ("modelcases", "llama_tiny_q4km", None, 8, 12, None),
    "llama_gqa_q5km": ("modelcases", "llama_gqa_q5km", None, 8, 12, None),
    "falcon_tiny_q5km": ("modelcases", "falcon_tiny_q5km", None, 8, 12, None),
    "llama_wide_q4km": ("modelcases", "llama_wide_q4km", None, 8, 12, None),
    "llama_ff11008_q4km": ("shape", "llama_ff11008_q4km", 37, 8, 12, 96),
    "falcon_ff18432_q5km": ("shape", "falcon_ff18432_q5km", 37, 8, 12, 96),
    "llama_hd80_q4km": ("shape", "llama_hd80_q4km", 37, 8, 12, 96),
    "llama_gqa_q3km": ("q3k", "llama_gqa_q3km", None, 8, 12, None),
    "llama_tiny_q4km_c1024_p600": ("modelcases", "llama_tiny_q4km", 600, 512, 8, 1024),
    "norm_llama_tiny_q4km": ("norm", "llama_tiny_q4km", None, None, None, None),
    "norm_falcon_tiny_q5km": ("norm", "falcon_tiny_q5km", None, None, None, None),
}
UNPAIRED = {"llama_gqa_q3km"}   # Q3_K programs run one CTA per cluster in both processes


def _shapes():
    """The model cases of kind "shape": name -> (arch, shape, ftype)."""
    from ctransformers_b200 import synth
    L, F = synth.LlamaShape, synth.FalconShape
    return {
        # down input 43 blocks: rank 0 stages 22, the last 32 of its 704 groups of 16 in a second group per thread
        "llama_ff11008_q4km": ("llama", L(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=11008, n_layer=2, n_ctx_train=256), "Q4_K_M"),
        # down input 72 blocks: 36 per rank, 576 groups of 16, LayerNorm on the 256-wide inputs
        "falcon_ff18432_q5km": ("falcon", F(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=1, n_ff=18432, n_layer=2, n_ctx_train=256), "Q5_K_M"),
        # heads of 80: k_step's build for other head sizes
        "llama_hd80_q4km": ("llama", L(n_vocab=1024, n_embd=1280, n_head=16, n_head_kv=4, n_ff=1536, n_layer=2, n_ctx_train=256), "Q4_K_M"),
    }
NORM_KS = [256, 512, 1024, 4096, 4608, 8192, 11008]   # test_norm_order.KS that the step kernel takes


def _build(run, directory):
    """(model path, context, prompt) of a run; the model file is written in the parent process, once for both launch shapes."""
    import modelcases
    kind, case, n_prompt, _, _, ctx = RUNS[run]
    if kind == "q3k":
        import q3k_refs
        path, c = q3k_refs.build_model(case, directory)
        return path, c, q3k_refs.prompt_for(case)
    if kind == "norm":
        path, c = modelcases.build_norm_order(case, directory)
        return path, c, None
    if kind == "shape":
        from ctransformers_b200 import synth
        arch, shape, ftype = _shapes()[case]
        path = Path(directory) / f"{case}.gguf"
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=11)
        ids = np.random.default_rng(5).integers(259 if arch == "llama" else 0, shape.n_vocab, n_prompt).tolist()
        if arch == "llama":
            ids[0] = 1
        return path, ctx, ids
    path, c = modelcases.build(case, directory)
    prompt = modelcases.prompt_for(case) if n_prompt is None else modelcases.seeded_prompt(case, n_prompt)
    return path, ctx or c, prompt


def _worker(spec_file, out_file):
    """Runs in a child process: every run of the spec with this process's launch shape; writes the results as one .npz."""
    sys.path[:0] = [str(ROOT), str(HERE)]
    from ctransformers_b200 import AutoModelForCausalLM
    spec = json.loads(Path(spec_file).read_text())
    out = {}
    for run, (path, ctx, prompt) in spec["models"].items():
        kind, case, _, bs, n_new, _ = RUNS[run]
        llm = AutoModelForCausalLM.from_pretrained(path, context_length=ctx)
        out[f"{run}/cluster"] = np.array([llm.ctb_llm_step_cluster()])
        if kind == "norm":
            import modelcases
            states, toks = modelcases.norm_order_llm_run(llm, case)
            out[f"{run}/logits"] = np.stack([s[0] for s in states])
            out[f"{run}/embd"] = np.stack([s[1] for s in states])
            out[f"{run}/tokens"] = np.array(toks)
            continue
        llm.eval(prompt, batch_size=bs)
        logits, embd, toks = [np.array(llm.logits, np.float32)], [np.array(llm.embeddings, np.float32)], []
        for _ in range(n_new):
            toks.append(int(llm.sample(top_k=1, repetition_penalty=1.0, seed=0)))
            llm.eval([toks[-1]])
            logits.append(np.array(llm.logits, np.float32))
            embd.append(np.array(llm.embeddings, np.float32))
        out[f"{run}/logits"], out[f"{run}/embd"], out[f"{run}/tokens"] = np.stack(logits), np.stack(embd), np.array(toks)
    if spec["norm_rows"]:   # one mat-vec phase of the step kernel, the normalised vector of the planted rows
        import ctypes as C
        import refs
        from ctransformers_b200.lib import load_library
        lib = load_library()
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        for mode in (1, 2):
            for k in NORM_KS:
                out[f"norm_path_cluster/{k}"] = np.array([lib.ctb_norm_path_cluster(k)])
                rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
                got = np.zeros_like(rows)
                for i in range(rows.shape[0]):
                    assert lib.ctb_norm_path(1, mode, p(rows[i]), p(w), p(b) if mode == 2 else None, p(got[i]), k, refs.NORM_ORDER_EPS) == 0
                out[f"norm_path/{mode}/{k}"] = got
    np.savez(out_file, **out)


def _run_shape(tmp, cluster, spec):
    """The spec's runs in a child process with CTB_ST_CLUSTER=cluster ("0" or "1"); returns the child's results."""
    spec_file, out_file = tmp / "spec.json", tmp / f"out_{cluster}.npz"
    spec_file.write_text(json.dumps(spec))
    env = dict(os.environ, CTB_ST_CLUSTER=cluster)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), str(Path(__file__).resolve()), str(spec_file), str(out_file)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"CTB_ST_CLUSTER={cluster} run failed:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"
    return dict(np.load(out_file))


@pytest.fixture(scope="module")
def both_shapes(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("cluster_stage")
    models = {}
    for run in RUNS:
        path, ctx, prompt = _build(run, tmp)
        models[run] = (str(path), ctx, prompt)
    spec = {"models": models, "norm_rows": True}
    return _run_shape(tmp, "0", spec), _run_shape(tmp, "1", spec)


@pytest.mark.gpu
def test_launch_shapes(both_shapes):
    """CTB_ST_CLUSTER=0 keeps one CTA per cluster; otherwise an H100 (132 SMs, every TPC two SMs) runs the step kernel in pairs,
    except for programs with Q3_K matrices.  The one-phase programs of ctb_norm_path are paired too."""
    single, paired = both_shapes
    for run in RUNS:
        assert int(single[f"{run}/cluster"][0]) == 1, run
        assert int(paired[f"{run}/cluster"][0]) == (1 if run in UNPAIRED else 2), run
    for k in NORM_KS:
        assert int(single[f"norm_path_cluster/{k}"][0]) == 1 and int(paired[f"norm_path_cluster/{k}"][0]) == 2, k


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_paired_staging_same_bits(both_shapes, run):
    single, paired = both_shapes
    for what in ("logits", "embd"):
        a, b = single[f"{run}/{what}"], paired[f"{run}/{what}"]
        assert a.shape == b.shape
        bad = (a.view(np.uint32) != b.view(np.uint32)).any(axis=1)
        assert not bad.any(), f"{run}: {what} of states {np.flatnonzero(bad).tolist()} of {len(bad)} differ between the launch shapes"
    assert single[f"{run}/tokens"].tolist() == paired[f"{run}/tokens"].tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("k", NORM_KS)
@pytest.mark.parametrize("mode", [1, 2])
def test_paired_norm_planted_rows(both_shapes, mode, k):
    """The normalised vector the step kernel writes for rows whose fp64 sum order shows: both ranks of the first pair write
    their blocks of it.  (test_norm_order_gpu compares the default launch shape with the oracle.)"""
    single, paired = both_shapes
    a, b = single[f"norm_path/{mode}/{k}"], paired[f"norm_path/{mode}/{k}"]
    bad = (a.view(np.uint32) != b.view(np.uint32)).any(axis=1)
    assert not bad.any(), f"rows {np.flatnonzero(bad).tolist()} of {len(bad)} differ"


if __name__ == "__main__":
    _worker(sys.argv[1], sys.argv[2])
