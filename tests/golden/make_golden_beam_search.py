"""Writes the beam search goldens from the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built by oracle/Makefile where
the reference sources are available):  python tests/golden/make_golden_beam_search.py

For every case of tests/beam_search_cases.py this evaluates the prompt through llama.cpp's C API (the context parameters of
ctransformers' llama_llm::Load, models/llms/llama.cc:87-103, chunked as LLM::BatchEval chunks at batch size 8), then calls
llama_beam_search (models/ggml/llama.cpp:4560-4571) with a callback that restates the one of examples/beam_search: a beam whose last
token is EOS is marked eob, and the common prefix is collected into the response.

  beam_search_runs.npz  per case key:
    <key>_response  the collected tokens (int32)
    <key>_p         the final beam's p as float32 bits (uint32)
    <key>_states    SHA-256 of every callback's beam state (beam_search_cases.state_digest), in call order

The generator asserts that the small-vocabulary cases mark eob beams and end runs on an eob top beam before n_predict.
"""
import ctypes as C
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import beam_search_cases as B  # noqa: E402
from make_golden_logits_all import reference  # noqa: E402


class BeamView(C.Structure):
    """struct llama_beam_view, models/ggml/llama.h:480-485"""
    _fields_ = [("tokens", C.POINTER(C.c_int)), ("n_tokens", C.c_size_t), ("p", C.c_float), ("eob", C.c_bool)]


class BeamsState(C.Structure):
    """struct llama_beams_state, models/ggml/llama.h:490-495"""
    _fields_ = [("beam_views", C.POINTER(BeamView)), ("n_beams", C.c_size_t), ("common_prefix_length", C.c_size_t), ("last_call", C.c_bool)]


CALLBACK = C.CFUNCTYPE(None, C.c_void_p, BeamsState)


def run(r, path, n_ctx, prompt, n_beams, n_predict, eos):
    p = r.llama_context_default_params()
    p.embedding, p.n_ctx, p.n_gpu_layers, p.use_mmap, p.use_mlock = True, n_ctx, 0, True, False
    model = r.llama_load_model_from_file(str(path).encode(), p)
    ctx = r.llama_new_context_with_model(model, p)
    assert model and ctx
    n_past = 0
    for start in range(0, len(prompt), B.BATCH_SIZE):
        chunk = prompt[start:start + B.BATCH_SIZE]
        assert r.llama_eval(ctx, (C.c_int * len(chunk))(*chunk), len(chunk), n_past, 4) == 0
        n_past += len(chunk)
    response, states = [], []
    stats = {"eob_marked": 0, "top_eob_stop": 0}

    def cb(_, st):
        views = [st.beam_views[i] for i in range(st.n_beams)]
        for v in views:
            if not v.eob and v.n_tokens and v.tokens[v.n_tokens - 1] == eos:
                v.eob = True
        stats["eob_marked"] += sum(v.eob for v in views)
        beams = [B.Beam([v.tokens[j] for j in range(v.n_tokens)], v.p, v.eob) for v in views]
        n = st.common_prefix_length
        response.extend(beams[0].tokens[:n])
        states.append(B.state_digest(beams, n, st.last_call))
        if st.last_call:
            stats["final_p"] = beams[0].p
    fn = CALLBACK(cb)
    r.llama_beam_search.argtypes = [C.c_void_p, CALLBACK, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
    r.llama_beam_search(ctx, fn, None, n_beams, n_past, n_predict, 4)
    r.llama_free(ctx)
    r.llama_free_model(model)
    return response, stats["final_p"], states, stats


def main():
    r = reference()
    out = {}
    small = {"eob_marked": 0, "top_eob_stop": 0}
    with tempfile.TemporaryDirectory() as tmp:
        for key, (name, prompt, nb, n_predict) in B.cases().items():
            path, n_ctx = B.build(name, tmp)
            response, p, states, stats = run(r, path, n_ctx, prompt, nb, n_predict, B.eos_of(name))
            out[f"{key}_response"] = np.array(response, np.int32)
            out[f"{key}_p"] = np.array([B.p_bits(p)], np.uint32)
            out[f"{key}_states"] = np.array(states)
            if name == B.SMALL:
                small["eob_marked"] += stats["eob_marked"]
                small["top_eob_stop"] += int(len(response) < n_predict and bool(response) and response[-1] == B.eos_of(name))
            print(key, len(states), "steps, response", len(response), flush=True)
    assert small["eob_marked"] > 0 and small["top_eob_stop"] > 0, small
    np.savez_compressed(HERE / "beam_search_runs.npz", **out)


if __name__ == "__main__":
    main()
