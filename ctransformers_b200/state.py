"""Sequence states (include/ctransformers_b200.h ctb_state_header): what a sequence has evaluated — its tokens, its K / V cache at
positions [0, n_past) and the results of its last eval — as one blob.  LLM.load_state and MultiLLM.restore take it back in any
handle of the same model file, whatever its context length or slot count, so a shared prompt is evaluated once and a
conversation can leave the GPU between turns."""
import ctypes as C
from array import array
from typing import Callable, List, Sequence

from .lib import StateHeader


class SequenceState:
    """A saved sequence: `tokens` (n_past = len(tokens)) and `data`, the library's blob, which holds the tokens too.  Picklable."""

    def __init__(self, tokens: Sequence[int], data):
        self.tokens: List[int] = list(tokens)
        self.data = data

    @property
    def n_past(self) -> int:
        return len(self.tokens)

    def header(self, lib) -> StateHeader:
        """The blob's header, checked by the library (ctb_state_info); ValueError when the blob is not a whole state."""
        h = StateHeader()
        if lib.ctb_state_info(_pointer(self.data), len(self.data), C.byref(h)) != 0:
            raise ValueError("Not a sequence state of this library (see the message above).")
        return h


def _pointer(data):
    return (C.c_char * len(data)).from_buffer(data) if isinstance(data, bytearray) else bytes(data)


def save(size_fn: Callable, save_fn: Callable, tokens: Sequence[int]) -> SequenceState:
    """size_fn(n_tokens) -> bytes; save_fn(tokens, n_tokens, buf, cap) -> 0 (ctb_llm_* / ctb_multi_* with the handle bound)."""
    tokens = list(tokens)
    n = len(tokens)
    size = size_fn(n)
    if size == 0:
        raise RuntimeError(f"No state of {n} tokens: the context holds at most the context length.")
    data = bytearray(size)
    if save_fn((C.c_int * max(n, 1))(*tokens), n, (C.c_char * size).from_buffer(data), size) != 0:
        raise RuntimeError("Failed to save the state.")
    return SequenceState(tokens, data)


def restore(lib, state: SequenceState, load_fn: Callable) -> List[int]:
    """load_fn(buf, size) -> 0.  Returns the tokens the handle has evaluated afterwards."""
    h = state.header(lib)
    held = array("i", bytes(memoryview(state.data)[C.sizeof(StateHeader): C.sizeof(StateHeader) + 4 * h.n_tokens])).tolist()
    if held != state.tokens:
        raise ValueError("The state's tokens are not the ones its blob holds.")
    if load_fn(_pointer(state.data), len(state.data)) != 0:
        raise RuntimeError("Failed to restore the state (see the message above).")
    return list(state.tokens)
