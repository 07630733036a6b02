"""Grammar-constrained sampling (include/ctransformers_b200.h ctb_grammar_*): grammars in the GBNF text format of llama.cpp's
grammar_parser::parse, and the state llama_sample_grammar / llama_grammar_accept_token work on.

    g = Grammar('root ::= "yes" | "no"')
    tokens = list(llm.generate(prompt_tokens, grammar=g))      # every token allowed by the grammar; ends at EOS

A state belongs to no model: accept(model, token) takes the pieces from the LLM or MultiLLM given, and sampling with a state
masks that model's vocabulary (on the GPU: csrc/grammar_gpu.cuh)."""
import ctypes as C
from typing import List, Optional, Tuple

from .lib import load_library


class Grammar:
    """A parsed grammar.  Raises ValueError with the parser's message and byte position for text the reference parser refuses
    (a syntax error), a grammar without `root`, a rule that is referenced but never defined, and left recursion."""

    def __init__(self, text: str, *, lib: Optional[str] = None):
        self._lib, self._g = load_library(lib), None
        self.text = text
        err, pos = C.create_string_buffer(512), C.c_long(-1)
        g = self._lib.ctb_grammar_parse(text.encode(), err, len(err), C.byref(pos))
        if not g:
            raise ValueError(f"grammar refused at byte {pos.value}: {err.value.decode(errors='replace')}")
        self._g = g

    @property
    def rules(self) -> List[List[Tuple[int, int]]]:
        """Every rule's elements as (type, value) pairs (llama_grammar_element), the END that closes it included."""
        info = (C.c_int * 3)()
        self._lib.ctb_grammar_info(self._g, info)
        n_rules, n_elems = info[0], info[1]
        off, elems = (C.c_int * (n_rules + 1))(), (C.c_uint * max(2 * n_elems, 1))()
        self._lib.ctb_grammar_rules(self._g, off, elems)
        return [[(elems[2 * e], elems[2 * e + 1]) for e in range(off[r], off[r + 1])] for r in range(n_rules)]

    @property
    def symbol_ids(self) -> dict:
        """name -> rule id, as the reference parser's parse_state.symbol_ids (generated rules are `name_N`)."""
        info = (C.c_int * 3)()
        self._lib.ctb_grammar_info(self._g, info)
        out, buf, rid = {}, C.create_string_buffer(4096), C.c_uint()
        for i in range(info[2]):
            n = self._lib.ctb_grammar_symbol(self._g, i, buf, len(buf), C.byref(rid))
            out[buf.raw[:n].decode()] = rid.value
        return out

    def start(self) -> "GrammarState":
        """The state before any token: llama_grammar_init at `root`."""
        return GrammarState(self._lib, self._lib.ctb_grammar_start(self._g))

    def __del__(self):
        if self.__dict__.get("_g"):
            self._lib.ctb_grammar_free(self._g)
            self._g = None


def as_state(grammar) -> "GrammarState":
    """A fresh state for a Grammar or GBNF text; a GrammarState as it is."""
    if isinstance(grammar, GrammarState):
        return grammar
    return (grammar if isinstance(grammar, Grammar) else Grammar(grammar)).start()


class GrammarState:
    """The pushdown stacks of a grammar and the partial UTF-8 sequence of the tokens accepted so far."""

    def __init__(self, lib, handle):
        if not handle:
            raise RuntimeError("Failed to create a grammar state.")
        self._lib, self._s = lib, handle

    def accept(self, model, token: int) -> None:
        """Advances past `token` (llama_grammar_accept_token with model's piece).  A token the state does not allow, or EOS
        where no stack is empty, raises ValueError and leaves the state as it was."""
        if hasattr(model, "_m"):
            rc = self._lib.ctb_multi_grammar_accept(model._m, self._s, int(token))
        else:
            rc = self._lib.ctb_llm_grammar_accept(model._llm, self._s, int(token))
        if rc != 0:
            raise ValueError(f"the grammar does not allow token {token} here")

    def accept_piece(self, piece: bytes, *, eos: bool = False) -> None:
        """accept with the token's piece given (eos=True: the end-of-sequence token)."""
        if self._lib.ctb_grammar_accept_piece(self._s, piece, len(piece), int(eos)) != 0:
            raise ValueError("the grammar does not allow this piece here" if not eos else "the grammar does not allow the end here")

    def copy(self) -> "GrammarState":
        return GrammarState(self._lib, self._lib.ctb_grammar_state_copy(self._s))

    @property
    def allowed_eos(self) -> bool:
        """Whether some stack is empty: the grammar allows the end of the sequence here."""
        return bool(self._lib.ctb_grammar_state_eos_ok(self._s))

    @property
    def stacks(self) -> Tuple[List[List[int]], Tuple[int, int]]:
        """The stacks (element indices into the grammar's rules laid end to end, bottom first, in the reference's order) and the
        partial UTF-8 sequence (value, bytes remaining; -1: an invalid sequence)."""
        part = (C.c_int * 2)()
        n = self._lib.ctb_grammar_state_stacks(self._s, None, 0, part)
        buf = (C.c_int * max(-n, 1))()
        n = self._lib.ctb_grammar_state_stacks(self._s, buf, max(-n, 0), part)
        out, i = [], 0
        while i < n:
            out.append(list(buf[i + 1:i + 1 + buf[i]]))
            i += 1 + buf[i]
        return out, (part[0], part[1])

    def mask_pieces(self, pieces: List[bytes], eos: int):
        """The host mask over the given pieces (piece t of token t): a bool array, True where llama_sample_grammar leaves the
        logit finite."""
        import numpy as np
        off = (C.c_int * (len(pieces) + 1))(*np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(int).tolist())
        out = np.zeros(len(pieces), np.uint8)
        if self._lib.ctb_grammar_mask_pieces(self._s, len(pieces), off, b"".join(pieces), eos, out.ctypes.data) != 0:
            raise RuntimeError("grammar mask failed")
        return out.astype(bool)

    def __del__(self):
        if self.__dict__.get("_s"):
            self._lib.ctb_grammar_state_free(self._s)
            self._s = None
