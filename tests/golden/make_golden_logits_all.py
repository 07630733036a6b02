"""Writes the logits_all golden digests from the UNMODIFIED reference (oracle/_ref/libctransformers_ref.so, built by oracle/Makefile
where the reference sources are available):  python tests/golden/make_golden_logits_all.py

The reference's llama.cpp keeps the logits row of every token of a llama_eval call when its context is created with the flag
logits_all (models/ggml/llama.cpp:2949-2960); ctransformers never sets it.  This script drives the reference build through
llama.cpp's own C API (llama_context_params bound by ctypes from models/ggml/llama.h), with the context parameters ctransformers'
llama_llm::Load uses (models/llms/llama.cc:87-103) plus logits_all, and with the chunking and n_past clamp of LLM::BatchEval
(models/llm.h:40-54, 124-137).

  logits_all_runs.npz  for every model case of modelcases / q3k_refs / q41_q51_refs / head_dims_refs (not their 7B- / 3B-shaped
                       cases) at batch sizes 8, 64 and 5, and for one eval that overflows the context (n_past clamped):
                         <key>_chunks     SHA-256 of each llama_eval call's row block (n x n_vocab float32), in call order
                         <key>_first_row  the first token's row, <key>_last_row the last token's (for diagnosis)

The files of the other generators are not touched.
"""
import ctypes as C
import hashlib
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import logits_all_cases as LA  # noqa: E402
import refs  # noqa: E402


class ContextParams(C.Structure):
    """struct llama_context_params, models/ggml/llama.h:125-152."""
    _fields_ = [("seed", C.c_uint32), ("n_ctx", C.c_int32), ("n_batch", C.c_int32), ("n_gpu_layers", C.c_int32), ("main_gpu", C.c_int32),
                ("tensor_split", C.POINTER(C.c_float)), ("rope_freq_base", C.c_float), ("rope_freq_scale", C.c_float),
                ("progress_callback", C.c_void_p), ("progress_callback_user_data", C.c_void_p),
                ("low_vram", C.c_bool), ("mul_mat_q", C.c_bool), ("f16_kv", C.c_bool), ("logits_all", C.c_bool), ("vocab_only", C.c_bool),
                ("use_mmap", C.c_bool), ("use_mlock", C.c_bool), ("embedding", C.c_bool)]


def reference():
    r = C.CDLL(str(refs.REF_SO))
    r.llama_context_default_params.restype = ContextParams
    r.llama_backend_init.argtypes = [C.c_bool]
    r.llama_load_model_from_file.restype = C.c_void_p
    r.llama_load_model_from_file.argtypes = [C.c_char_p, ContextParams]
    r.llama_new_context_with_model.restype = C.c_void_p
    r.llama_new_context_with_model.argtypes = [C.c_void_p, ContextParams]
    r.llama_eval.restype = C.c_int
    r.llama_eval.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int]
    r.llama_get_logits.restype = C.POINTER(C.c_float)
    r.llama_get_logits.argtypes = [C.c_void_p]
    r.llama_free.argtypes = [C.c_void_p]
    r.llama_free_model.argtypes = [C.c_void_p]
    r.llama_backend_init(False)
    return r


class RefContext:
    def __init__(self, r, path, n_ctx, n_vocab):
        self.r, self.n_ctx, self.n_vocab, self.n_past = r, n_ctx, n_vocab, 0
        p = r.llama_context_default_params()
        p.embedding, p.n_ctx, p.n_gpu_layers, p.use_mmap, p.use_mlock = True, n_ctx, 0, True, False   # llama.cc:87-96
        p.logits_all = True
        self.model = r.llama_load_model_from_file(str(path).encode(), p)
        self.ctx = r.llama_new_context_with_model(self.model, p)
        assert self.model and self.ctx

    def batch_eval(self, tokens, batch_size):
        """LLM::BatchEval: one llama_eval per chunk; returns each chunk's row block."""
        bs = min(self.n_ctx, batch_size)
        blocks = []
        for start in range(0, len(tokens), bs):
            chunk = tokens[start:start + bs]
            past = min(self.n_ctx - len(chunk), self.n_past)
            arr = (C.c_int * len(chunk))(*chunk)
            assert self.r.llama_eval(self.ctx, arr, len(chunk), past, 4) == 0
            rows = np.ctypeslib.as_array(self.r.llama_get_logits(self.ctx), (len(chunk) * self.n_vocab,))
            blocks.append(rows.reshape(len(chunk), self.n_vocab).copy())
            self.n_past += len(chunk)
        return blocks

    def close(self):
        self.r.llama_free(self.ctx)
        self.r.llama_free_model(self.model)


def main():
    r = reference()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for key, (name, calls) in LA.runs().items():
            path, ctx = LA.build(name, tmp)
            ref = RefContext(r, path, ctx, LA.n_vocab(name))
            blocks = []
            for toks, bs in calls:
                blocks += ref.batch_eval(toks, bs)
            ref.close()
            out[f"{key}_chunks"] = np.array([hashlib.sha256(np.ascontiguousarray(b).tobytes()).hexdigest() for b in blocks])
            out[f"{key}_first_row"] = blocks[0][0]
            out[f"{key}_last_row"] = blocks[-1][-1]
            print(key, len(blocks), "chunks", flush=True)
    np.savez_compressed(HERE / "logits_all_runs.npz", **out)


if __name__ == "__main__":
    main()
