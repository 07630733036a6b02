"""Locate and bind libctransformers.so (the H100 build).

Mirror of the reference's FFI layer (ctransformers/lib.py:9-73 `find_library`, ctransformers/llm.py:117-208
`load_library`): same 17 prototypes, plus the additive ``ctb_*`` entry points of include/ctransformers_b200.h.
There is exactly one library flavour here — the in-tree sm_90a build — and no fallback: a missing library is
an error, never a silent switch to another code path.
"""
import ctypes as C
from pathlib import Path
from typing import Optional

LIB_DIR = Path(__file__).resolve().parent / "lib"
LIB_NAME = "libctransformers.so"


class ConfigStruct(C.Structure):
    """By-value argument of ctransformers_llm_create (reference: models/llm.h:6-11)."""
    _fields_ = [("context_length", C.c_int), ("gpu_layers", C.c_int), ("mmap", C.c_bool), ("mlock", C.c_bool)]


def find_library(path: Optional[str] = None) -> str:
    """An explicit path wins (like the reference, which returns unknown strings verbatim); otherwise the in-tree build."""
    if path:
        return str(path)
    lib = LIB_DIR / LIB_NAME
    if not lib.is_file():
        raise OSError(
            f"{lib} has not been built. Build it with `python -m ctransformers_b200.build` "
            "(needs nvcc; compiles for sm_90a). There is no CPU fallback library."
        )
    return str(lib)


_P = C.c_void_p
_IP = C.POINTER(C.c_int)
_FP = C.POINTER(C.c_float)
_DP = C.POINTER(C.c_double)

# name -> (restype, argtypes); part 1 = the reference FFI (models/llm.cc:32-138)
PROTOTYPES = {
    "ctransformers_llm_create": (_P, [C.c_char_p, C.c_char_p, ConfigStruct]),
    "ctransformers_llm_delete": (None, [_P]),
    "ctransformers_llm_tokenize": (C.c_int, [_P, C.c_char_p, C.c_bool, _IP]),
    "ctransformers_llm_detokenize": (C.c_char_p, [_P, C.c_int]),
    "ctransformers_llm_is_eos_token": (C.c_bool, [_P, C.c_int]),
    "ctransformers_llm_eos_token_id": (C.c_int, [_P]),
    "ctransformers_llm_bos_token_id": (C.c_int, [_P]),
    "ctransformers_llm_vocab_size": (C.c_int, [_P]),
    "ctransformers_llm_context_length": (C.c_int, [_P]),
    "ctransformers_llm_architecture": (C.c_char_p, [_P]),
    "ctransformers_llm_batch_eval": (C.c_bool, [_P, _IP, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ctransformers_llm_logits_data": (_FP, [_P]),
    "ctransformers_llm_logits_size": (C.c_int, [_P]),
    "ctransformers_llm_embeddings_data": (_FP, [_P]),
    "ctransformers_llm_embeddings_size": (C.c_int, [_P]),
    "ctransformers_llm_sample": (C.c_int, [_P, _IP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]),
    "ctransformers_llm_reset": (None, [_P]),
}
# part 2 = additive entry points
EXTRA_PROTOTYPES = {
    "ctb_abi_version": (C.c_int, []),
    "ctb_llm_last_eval_ms": (C.c_double, [_P]),
    "ctb_llm_launches_per_token": (C.c_long, [_P]),
    "ctb_llm_speculative_hits": (C.c_long, [_P]),
    "ctb_llm_weight_bytes_per_token": (C.c_ulonglong, [_P]),
    "ctb_llm_trace_step": (C.c_long, [_P, C.c_int, C.c_int, C.POINTER(C.c_ulonglong), C.c_long]),
    "ctb_llm_load_ms": (C.c_double, [_P]),
    "ctb_llm_device_samples": (C.c_long, [_P]),
    "ctb_llm_set_stream": (None, [_P, C.c_void_p]),
    "ctb_tp_unique_id": (C.c_int, [_P, C.c_int]),
    "ctb_llm_create_tp": (_P, [C.c_char_p, C.c_char_p, ConfigStruct, C.c_int, C.c_int, _P]),
    "ctb_tp_shard": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _IP]),
    "ctb_llm_decode_greedy": (C.c_double, [_P, C.c_int, C.c_int, C.c_int, _IP]),
    "ctb_llm_profile_step": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_double), _IP]),
    "ctb_llm_time_matvec_only": (C.c_double, [_P, C.c_int, C.POINTER(C.c_long)]),
    "ctb_llm_time_matvec_kinds": (C.c_double, [_P, C.c_int, C.POINTER(C.c_long), C.c_uint]),
    "ctb_mul_mat": (C.c_int, [C.c_int, _P, _P, _P, C.c_int, C.c_int, C.c_int]),
    "ctb_quantize_row_q8_K": (C.c_int, [_P, _P, C.c_int]),
    "ctb_quantize_row_q8_0": (C.c_int, [_P, _P, C.c_int]),
    "ctb_quantize_row_q8_1": (C.c_int, [_P, _P, C.c_int]),
    "ctb_norm": (C.c_int, [C.c_int, _P, _P, _P, _P, C.c_int, C.c_float]),
    "ctb_norm_path": (C.c_int, [C.c_int, C.c_int, _P, _P, _P, _P, C.c_int, C.c_float]),
    "ctb_rope": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float]),
    "ctb_attention": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "ctb_attention_path": (C.c_int, [C.c_int, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int,
                                     C.c_float, C.c_float]),
    "ctb_prefill_mul_mat": (C.c_int, [C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, C.c_float, _P, _P, _P, _P, C.c_int,
                                      C.c_int, _P]),
    "ctb_llm_paths": (C.c_long, [_P, _IP, C.c_int]),
    "ctb_ffn_gate": (C.c_int, [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int]),
    "ctb_matvec_partition": (C.c_int, [_IP, _IP, C.c_int, C.c_int, C.c_int, _IP, _IP]),
    "ctb_get_row": (C.c_int, [C.c_int, _P, C.c_int, C.c_int, C.c_int, _P]),
    "ctb_argmax_path": (C.c_int, [C.c_int, _P, C.c_int, _IP]),
    "ctb_sample_topk": (C.c_int, [_P, C.c_int, _IP, C.c_int, C.c_float, C.c_int, _IP, _P]),
    "ctb_sample_device": (C.c_int, [_P, C.c_int, _IP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, _IP]),
    "ctb_sample_topk_rows": (C.c_int, [_P, C.c_int, C.c_int, _IP, _IP, _FP, _IP, _IP, _IP, _FP]),
    "ctb_sample_device_rows": (C.c_int, [_P, C.c_int, C.c_int, _IP, _IP, _IP, _FP, _FP, _FP, _IP, _IP, _IP]),
    "ctb_vocab_load": (_P, [C.c_char_p]),
    "ctb_vocab_free": (None, [_P]),
    "ctb_vocab_size": (C.c_int, [_P]),
    "ctb_vocab_tokenize": (C.c_int, [_P, C.c_char_p, C.c_bool, _IP, C.c_int]),
    "ctb_vocab_piece": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_int]),
    "ctb_sample": (C.c_int, [_FP, C.c_int, _IP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]),
    "ctb_multi_create": (_P, [C.c_char_p, C.c_char_p, ConfigStruct, C.c_int]),
    "ctb_multi_delete": (None, [_P]),
    "ctb_multi_info": (C.c_int, [_P, _IP]),
    "ctb_multi_eval": (C.c_bool, [_P, C.c_int, _IP, _IP, _IP, _IP, C.c_int]),
    "ctb_multi_logits": (_FP, [_P, C.c_int]),
    "ctb_multi_embeddings": (_FP, [_P, C.c_int]),
    "ctb_multi_greedy": (C.c_int, [_P, C.c_int, _IP, _IP]),
    "ctb_multi_sample": (C.c_int, [_P, C.c_int, _IP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]),
    "ctb_multi_sample_many": (C.c_int, [_P, C.c_int, _IP, _IP, _IP, _IP, _FP, _FP, _FP, _IP, _IP]),
    "ctb_multi_device_samples": (C.c_long, [_P]),
    "ctb_multi_reset": (C.c_int, [_P, C.c_int]),
    "ctb_multi_launches": (C.c_long, [_P]),
    "ctb_multi_last_eval_ms": (C.c_double, [_P]),
    "ctb_multi_pack": (C.c_int, [C.c_int, _IP, _IP, _IP, C.c_int, C.c_int, _IP, C.c_int]),
    "ctb_state_info": (C.c_int, [_P, C.c_size_t, _P]),
    "ctb_llm_state_size": (C.c_size_t, [_P, C.c_int]),
    "ctb_llm_save_state": (C.c_int, [_P, _IP, C.c_int, _P, C.c_size_t]),
    "ctb_llm_load_state": (C.c_int, [_P, _P, C.c_size_t]),
    "ctb_multi_state_size": (C.c_size_t, [_P, C.c_int]),
    "ctb_multi_save": (C.c_int, [_P, C.c_int, _IP, C.c_int, _P, C.c_size_t]),
    "ctb_multi_restore": (C.c_int, [_P, C.c_int, _P, C.c_size_t]),
    "ctb_multi_fork": (C.c_int, [_P, C.c_int, C.c_int, _IP]),
    "ctb_llm_batch_eval_rows": (C.c_int, [_P, _IP, C.c_int, C.c_int, C.c_int, _FP]),
    "ctb_llm_batch_eval_scored": (C.c_int, [_P, _IP, C.c_int, C.c_int, C.c_int, _IP, _DP, _IP]),
    "ctb_llm_score_last": (C.c_int, [_P, C.c_int, _DP, _IP]),
    "ctb_row_logprob": (C.c_int, [_P, C.c_int, C.c_int, _IP, _DP, _IP]),
    "ctb_multi_eval_rows": (C.c_int, [_P, C.c_int, _IP, _IP, _IP, _IP, C.c_int, _FP]),
    "ctb_multi_eval_scored": (C.c_int, [_P, C.c_int, _IP, _IP, _IP, _IP, C.c_int, _IP, _DP, _IP]),
    "ctb_beam_step": (C.c_int, [C.c_int, C.c_int, C.c_int, _FP, _P, _FP, C.c_int, _IP, _IP, _FP, _P]),
    "ctb_multi_reparent": (C.c_long, [_P, C.c_int, _IP, _IP, _IP, _IP]),
    "ctb_multi_beam_search": (C.c_int, [_P, C.c_int, _IP, _IP, C.c_int, C.c_int, C.c_int, _IP, _IP, _FP]),
    "ctb_multi_beam_stats": (C.c_int, [_P, _DP]),
    "ctb_grammar_parse": (_P, [C.c_char_p, C.c_char_p, C.c_int, C.POINTER(C.c_long)]),
    "ctb_grammar_free": (None, [_P]),
    "ctb_grammar_info": (C.c_int, [_P, _IP]),
    "ctb_grammar_rules": (C.c_int, [_P, _IP, C.POINTER(C.c_uint)]),
    "ctb_grammar_symbol": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_uint)]),
    "ctb_grammar_start": (_P, [_P]),
    "ctb_grammar_state_copy": (_P, [_P]),
    "ctb_grammar_state_free": (None, [_P]),
    "ctb_grammar_state_eos_ok": (C.c_int, [_P]),
    "ctb_grammar_state_stacks": (C.c_int, [_P, _IP, C.c_int, _IP]),
    "ctb_grammar_accept_piece": (C.c_int, [_P, C.c_char_p, C.c_int, C.c_int]),
    "ctb_llm_grammar_accept": (C.c_int, [_P, _P, C.c_int]),
    "ctb_multi_grammar_accept": (C.c_int, [_P, _P, C.c_int]),
    "ctb_grammar_mask_pieces": (C.c_int, [_P, C.c_int, _IP, C.c_char_p, C.c_int, _P]),
    "ctb_llm_grammar_mask": (C.c_int, [_P, _P, _P]),
    "ctb_multi_grammar_mask": (C.c_int, [_P, C.c_int, _P, _P]),
    "ctb_llm_sample_grammar": (C.c_int, [_P, _IP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, _P]),
    "ctb_multi_sample_grammar_many": (C.c_int, [_P, C.c_int, _IP, _IP, _IP, _IP, _FP, _FP, _FP, _IP, C.POINTER(_P), _IP]),
    "ctb_llm_grammar_paths": (C.c_int, [_P, C.POINTER(C.c_long)]),
    "ctb_multi_grammar_paths": (C.c_int, [_P, C.POINTER(C.c_long)]),
}


class StateHeader(C.Structure):
    """ctb_state_header (include/ctransformers_b200.h): the header of a sequence state."""
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("n_layer", C.c_int32), ("n_head_kv", C.c_int32), ("head_dim", C.c_int32),
                ("k_stride", C.c_int32), ("n_embd", C.c_int32), ("n_vocab", C.c_int32), ("n_tokens", C.c_int32), ("has_results", C.c_int32),
                ("fingerprint", C.c_uint64)]


def load_library(path: Optional[str] = None):
    lib = C.CDLL(find_library(path))
    for table, required in ((PROTOTYPES, True), (EXTRA_PROTOTYPES, False)):
        for name, (res, args) in table.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                if required:
                    raise OSError(f"{path or LIB_NAME} does not export '{name}'")
                continue  # a reference-built library has no ctb_* symbols; that is fine when passed via lib=
            fn.restype, fn.argtypes = res, args
    return lib
