"""Python surface over the C ABI — the H100 counterpart of ctransformers/llm.py (reference lines cited inline).

Same class names, method names, keyword arguments, defaults and error behaviour, so code written against
``ctransformers.LLM`` runs unchanged:  tokenize / detokenize / eval / sample / generate / __call__ / embed,
`Config`, the zero-copy writable `logits` view, prefix reuse in `prepare_inputs_for_generation`.
"""
import re
import warnings
from collections.abc import MutableSequence
from ctypes import POINTER, byref, c_double, c_float, c_int
from dataclasses import dataclass, fields
from functools import partial
from pathlib import Path
from typing import Generator, List, Optional, Sequence, Union

from . import state
from .lib import ConfigStruct, load_library
from .state import SequenceState

import logging

logger = logging.getLogger("ctransformers_b200")


@dataclass
class Config:
    """Defaults identical to the reference (ctransformers/llm.py:38-61)."""
    top_k: int = 40
    top_p: float = 0.95
    temperature: float = 0.8
    repetition_penalty: float = 1.1
    last_n_tokens: int = 64
    seed: int = -1
    batch_size: int = 8
    threads: int = -1
    max_new_tokens: int = 256
    stop: Optional[Sequence[str]] = None
    stream: bool = False
    reset: bool = True
    context_length: int = -1
    gpu_layers: int = 0
    mmap: bool = True
    mlock: bool = False

    def to_struct(self) -> ConfigStruct:
        return ConfigStruct(self.context_length, self.gpu_layers, self.mmap, self.mlock)


def _pick(*values):
    for v in values:
        if v is not None:
            return v
    return None


def is_gguf(path) -> bool:
    with open(path, "rb") as f:
        return f.read(4) == b"GGUF"


class Vector(MutableSequence):
    """List-like, in-place view of a C float array (reference: ctransformers/utils.py:13-43).  Writes go straight to the
    library-owned buffer, which is what lets callers edit `llm.logits` before `llm.sample()` (tests/test_model.py:10-16)."""

    def __init__(self, data, size):
        self._data, self._size = data, size

    def _at(self, i):
        if not isinstance(i, int):
            raise TypeError("list index must be integer")
        if not 0 <= i < self._size:
            raise IndexError("list index out of range")
        return i

    def __getitem__(self, i):
        return self._data[self._at(i)]

    def __setitem__(self, i, v):
        self._data[self._at(i)] = v

    def __len__(self):
        return self._size

    def __delitem__(self, i):
        raise NotImplementedError("This operation is not allowed.")

    def insert(self, i, v):
        raise NotImplementedError("This operation is not allowed.")


def _split_incomplete_utf8(seq: bytes):
    """Bytes up to the last character boundary, and the dangling tail (reference: utils.py:46-56)."""
    i = len(seq)
    while i > 0 and seq[i - 1] & 0x80:
        i -= 1
    return seq[:i], seq[i:]


def _check_ids(tokens: Sequence[int], n_vocab: int, what: str, lo: int = 0) -> List[int]:
    """tokens as a list of ints, each in [lo, n_vocab): what the library would refuse is refused here, with the culprit named."""
    ids = [int(t) for t in tokens]
    for i, t in enumerate(ids):
        if not lo <= t < n_vocab:
            raise ValueError(f"{what} {i} is {t}: out of range ({lo} .. {n_vocab - 1})")
    return ids


def _ints(values: Sequence[int]):
    return (c_int * max(len(values), 1))(*values)


class LLM:
    all_logits = None   # eval(..., logits_all=True): the rows of that eval's tokens

    def __init__(self, model_path: str, model_type: Optional[str] = None, *, config: Optional[Config] = None, lib: Optional[str] = None, tp=None):
        """Loads a GGUF model onto the GPU (reference: ctransformers/llm.py:212-259).
        tp = (rank, world, unique_id_bytes) loads this process's shard of the tensor-sharded mode (ctransformers_b200/tp.py;
        an extension: the reference has no multi-GPU path)."""
        self._config = config or Config()
        self._model_path, self._llm, self._lib, self._context = model_path, None, None, []
        if not Path(model_path).is_file():
            raise ValueError(f"Model path '{model_path}' doesn't exist.")
        if not model_type:
            if not is_gguf(model_path):
                raise ValueError("Unable to detect model type. Please specify a model type using:\n\n"
                                 "  AutoModelForCausalLM.from_pretrained(..., model_type='...')\n\n")
            model_type = "gguf"
        self._lib = load_library(lib)
        if tp is not None and tp[1] > 1:
            rank, world, uid = tp
            self._llm = self._lib.ctb_llm_create_tp(model_path.encode(), model_type.encode(), self._config.to_struct(), rank, world, bytes(uid))
        else:
            self._llm = self._lib.ctransformers_llm_create(model_path.encode(), model_type.encode(), self._config.to_struct())
        if self._llm is None:
            raise RuntimeError(f"Failed to create LLM '{model_type}' from '{model_path}'.")
        self._model_type = self.ctransformers_llm_architecture().decode() or model_type

    # ---- properties (reference: llm.py:261-315)
    model_path = property(lambda self: self._model_path)
    model_type = property(lambda self: self._model_type)
    config = property(lambda self: self._config)
    eos_token_id = property(lambda self: self.ctransformers_llm_eos_token_id())
    bos_token_id = property(lambda self: self.ctransformers_llm_bos_token_id())
    pad_token_id = property(lambda self: self.ctransformers_llm_eos_token_id())
    vocab_size = property(lambda self: self.ctransformers_llm_vocab_size())
    context_length = property(lambda self: self.ctransformers_llm_context_length())

    @property
    def logits(self) -> List[float]:
        return Vector(self.ctransformers_llm_logits_data(), self.ctransformers_llm_logits_size())

    @property
    def embeddings(self) -> List[float]:
        return Vector(self.ctransformers_llm_embeddings_data(), self.ctransformers_llm_embeddings_size())

    def __getattr__(self, name):
        lib, llm = self.__dict__.get("_lib"), self.__dict__.get("_llm")
        if (name.startswith("ctransformers_llm_") or name.startswith("ctb_llm_")) and lib is not None and hasattr(lib, name):
            return partial(getattr(lib, name), llm)
        raise AttributeError(f"'LLM' object has no attribute '{name}'")

    # ---- text <-> tokens (reference: llm.py:323-365)
    def tokenize(self, text: str, add_bos_token: Optional[bool] = None) -> List[int]:
        if add_bos_token is None:
            add_bos_token = self.model_type == "llama"
        raw = text.encode()
        # The reference sizes this buffer len(text)+1 ints — characters, not bytes (llm.py:335-337) — although BOS + the SPM "▁"
        # prefix can yield len+2 tokens: its C side then writes one int past the end and the slice silently drops the last
        # token.  We return exactly what the reference returns (at most len(text)+1 tokens) but give the library room, so
        # nothing is written out of bounds.
        out = (c_int * (len(raw) + 8))()
        n = self.ctransformers_llm_tokenize(raw, add_bos_token, out)
        return out[: min(n, len(text) + 1)]

    def detokenize(self, tokens: Sequence[int], decode: bool = True) -> Union[str, bytes]:
        if isinstance(tokens, int):
            tokens = [tokens]
        data = b"".join(self.ctransformers_llm_detokenize(t) for t in tokens)
        if not decode:
            return data
        text = data.decode(errors="ignore")
        if list(tokens[:1]) == [self.bos_token_id] and text[:1] == " ":
            text = text[1:]
        return text

    def is_eos_token(self, token: int) -> bool:
        return self.ctransformers_llm_is_eos_token(token)

    # ---- eval / sample (reference: llm.py:379-455)
    def eval(self, tokens: Sequence[int], *, batch_size: Optional[int] = None, threads: Optional[int] = None, logits_all: bool = False) -> None:
        """logits_all=True (an extension; the reference's llama.cpp has the context flag, ctransformers never sets it) also keeps
        the logits of every evaluated token, not only the last one's: `all_logits` is then an (n, vocab_size) float32 array, row i
        bit-identical to the reference's row for tokens[i].  Everything else comes out as from an ordinary eval."""
        cfg = self._config
        batch_size, threads = _pick(batch_size, cfg.batch_size), _pick(threads, cfg.threads)
        n_past, n = len(self._context), len(tokens)
        if n_past + n > self.context_length:
            logger.warning(f"Number of tokens ({n_past + n}) exceeded maximum context length ({self.context_length}).")
        self.all_logits = None
        if logits_all:
            import numpy as np
            ids = _check_ids(tokens, self.vocab_size, "token")
            rows = np.empty((n, self.vocab_size), np.float32)
            if self._lib.ctb_llm_batch_eval_rows(self._llm, _ints(ids), n, n_past, batch_size, rows.ctypes.data_as(POINTER(c_float))) != 0:
                raise RuntimeError("Failed to evaluate tokens.")
            self._context.extend(ids)
            self.all_logits = rows
            return
        arr = (c_int * n)(*tokens)
        if not self.ctransformers_llm_batch_eval(arr, n, n_past, batch_size, threads):
            raise RuntimeError("Failed to evaluate tokens.")
        self._context.extend(arr)

    def score(self, tokens: Sequence[int], *, batch_size: Optional[int] = None):
        """Evaluates tokens after the current context and scores each of them under the logits that precede it.  Returns
        (logprob, greedy): float64 log-probabilities and bool flags "is the greedy pick" (sample(top_k=1)), one per token, reduced
        on the GPU (csrc/score_gpu.cuh defines both, NaN and infinite logits included).  Token 0 is scored from the last logits
        of the context; without a context nothing precedes it, and it gets NaN / False."""
        import numpy as np
        cfg = self._config
        batch_size = _pick(batch_size, cfg.batch_size)
        n_vocab = self.vocab_size
        ids = _check_ids(tokens, n_vocab, "token")
        n, n_past = len(ids), len(self._context)
        logprob, greedy = np.full(n, np.nan), np.zeros(n, bool)
        if n == 0:
            return logprob, greedy
        if n_past + n > self.context_length:
            logger.warning(f"Number of tokens ({n_past + n}) exceeded maximum context length ({self.context_length}).")
        if n_past:
            lp0, g0 = c_double(), c_int()
            if self._lib.ctb_llm_score_last(self._llm, ids[0], byref(lp0), byref(g0)) != 0:
                raise RuntimeError("Failed to score the first token against the last logits.")
            logprob[0], greedy[0] = lp0.value, bool(g0.value)
        lp, gr = np.zeros(n, np.float64), np.zeros(n, np.int32)
        if self._lib.ctb_llm_batch_eval_scored(self._llm, _ints(ids), n, n_past, batch_size, _ints(ids[1:] + [-1]),
                                               lp.ctypes.data_as(POINTER(c_double)), gr.ctypes.data_as(POINTER(c_int))) != 0:
            raise RuntimeError("Failed to evaluate tokens.")
        self._context.extend(ids)
        self.all_logits = None
        logprob[1:], greedy[1:] = lp[:-1], gr[:-1] != 0
        return logprob, greedy

    def perplexity(self, tokens: Sequence[int], *, batch_size: Optional[int] = None) -> float:
        """exp of the mean negative log-probability of the scored tokens (score: every token but a first one without context)."""
        import numpy as np
        had_context = bool(self._context)
        logprob, _ = self.score(tokens, batch_size=batch_size)
        scored = logprob if had_context else logprob[1:]
        if len(scored) == 0:
            raise ValueError("perplexity needs a scored token: give a context or at least two tokens")
        return float(np.exp(-np.mean(scored)))

    def sample(self, *, top_k=None, top_p=None, temperature=None, repetition_penalty=None, last_n_tokens=None, seed=None) -> int:
        cfg = self._config
        last_n = _pick(last_n_tokens, cfg.last_n_tokens)
        if last_n < 0:
            last_n = self.context_length
        recent = self._context[-last_n:]   # (last_n == 0 selects the whole context, exactly like the reference's slice, llm.py:443)
        arr = (c_int * len(recent))(*recent)
        return self.ctransformers_llm_sample(arr, len(recent), _pick(top_k, cfg.top_k), _pick(top_p, cfg.top_p),
                                             _pick(temperature, cfg.temperature), _pick(repetition_penalty, cfg.repetition_penalty),
                                             _pick(seed, cfg.seed))

    def save_state(self) -> SequenceState:
        """What this LLM has evaluated (its tokens, K / V cache and last results), for load_state here or in any LLM or MultiLLM
        of the same model file."""
        return state.save(partial(self._lib.ctb_llm_state_size, self._llm), partial(self._lib.ctb_llm_save_state, self._llm), self._context)

    def load_state(self, saved: SequenceState) -> None:
        """Continues from a saved state exactly as if its tokens had just been evaluated here."""
        self._context = state.restore(self._lib, saved, partial(self._lib.ctb_llm_load_state, self._llm))

    def reset(self) -> None:
        warnings.warn("`LLM.reset()` method is deprecated since 0.2.27. Please use high-level API.")
        self._context.clear()
        self.ctransformers_llm_reset()

    def __del__(self):
        if self.__dict__.get("_llm") is not None and self.__dict__.get("_lib") is not None:
            self._lib.ctransformers_llm_delete(self._llm)
            self._llm = None

    # ---- generation (reference: llm.py:470-664)
    def prepare_inputs_for_generation(self, tokens: Sequence[int], *, reset: Optional[bool] = None) -> Sequence[int]:
        """Drops the prefix that is already in the KV cache and truncates the context to it (llm.py:470-500)."""
        if not _pick(reset, self._config.reset):
            return tokens
        limit = min(len(tokens) - 1, len(self._context))   # always leave one token to evaluate
        keep = 0
        while keep < limit and tokens[keep] == self._context[keep]:
            keep += 1
        self._context = self._context[:keep]
        return tokens[keep:]

    def generate(self, tokens: Sequence[int], *, top_k=None, top_p=None, temperature=None, repetition_penalty=None, last_n_tokens=None,
                 seed=None, batch_size=None, threads=None, reset=None) -> Generator[int, None, None]:
        tokens = self.prepare_inputs_for_generation(tokens, reset=reset)
        self.eval(tokens, batch_size=batch_size, threads=threads)
        while True:
            token = self.sample(top_k=top_k, top_p=top_p, temperature=temperature, repetition_penalty=repetition_penalty,
                                last_n_tokens=last_n_tokens, seed=seed)
            self.eval([token], batch_size=batch_size, threads=threads)
            if self.is_eos_token(token):
                break
            yield token

    def _stream(self, prompt: str, *, max_new_tokens=None, stop=None, **sampling) -> Generator[str, None, None]:
        cfg = self._config
        max_new_tokens = _pick(max_new_tokens, cfg.max_new_tokens)
        stop = _pick(stop, cfg.stop) or []
        if isinstance(stop, str):
            stop = [stop]
        stop_re = re.compile("|".join(map(re.escape, stop)))
        text, pending, produced = "", b"", 0
        for token in self.generate(self.tokenize(prompt), **sampling):
            pending += self.detokenize([token], decode=False)
            whole, pending = _split_incomplete_utf8(pending)
            text += whole.decode(errors="ignore")
            if stop:
                hit = stop_re.search(text)
                if hit:
                    text = text[: hit.start()]
                    break
            # hold back the longest tail that could still grow into a stop sequence
            hold = 0
            for s in stop:
                for k in range(len(s), 0, -1):
                    if text.endswith(s[:k]):
                        hold = max(hold, k)
                        break
            cut = len(text) - hold
            if cut > 0:
                yield text[:cut]
                text = text[cut:]
            produced += 1
            if produced >= max_new_tokens:
                break
        if text:
            yield text

    def __call__(self, prompt: str, *, max_new_tokens=None, top_k=None, top_p=None, temperature=None, repetition_penalty=None,
                 last_n_tokens=None, seed=None, batch_size=None, threads=None, stop=None, stream=None, reset=None):
        pieces = self._stream(prompt, max_new_tokens=max_new_tokens, stop=stop, top_k=top_k, top_p=top_p, temperature=temperature,
                              repetition_penalty=repetition_penalty, last_n_tokens=last_n_tokens, seed=seed, batch_size=batch_size,
                              threads=threads, reset=reset)
        return pieces if _pick(stream, self._config.stream) else "".join(pieces)

    def embed(self, input: Union[str, Sequence[int]], *, batch_size=None, threads=None) -> List[float]:
        if isinstance(input, str):
            input = self.tokenize(input)
        input = self.prepare_inputs_for_generation(input, reset=True)
        self.eval(input, batch_size=batch_size, threads=threads)
        return list(self.embeddings)


CONFIG_FIELDS = {f.name for f in fields(Config)}
