"""Many independent sequences on one GPU (include/ctransformers_b200.h ctb_multi_*): every slot behaves like its own LLM with the
same config, bit for bit, while the slots listed in one eval share batched launches — one pass over the weights per launch of
up to 32 tokens instead of one per token of every sequence."""
from ctypes import POINTER, c_double, c_float, c_int
from pathlib import Path
from functools import partial
from typing import Dict, List, Optional, Sequence, Tuple

from .lib import load_library
from . import state
from .llm import Config, Vector, _check_ids, _ints, _pick, is_gguf
from .state import SequenceState


def per_slot(value, n: int, what: str) -> list:
    """`value` for each of n slots: one value for all of them, or a sequence holding one value per slot."""
    if isinstance(value, (str, bytes)) or not hasattr(value, "__len__"):
        return [value] * n
    values = list(value)
    if len(values) != n:
        raise ValueError(f"{what}: {len(values)} values for {n} slots")
    return values


def _flatten(lists: Sequence[Sequence[int]]) -> Tuple[List[int], List[int]]:
    """The lists concatenated, and the offsets where each starts (one more at the end): the library's (off, flat) form."""
    off, flat = [0], []
    for items in lists:
        flat.extend(items)
        off.append(len(flat))
    return off, flat


class MultiLLM:
    all_logits = None   # eval(..., logits_all=True): {slot: the rows of that slot's tokens}

    def __init__(self, model_path: str, model_type: Optional[str] = None, *, n_slots: int, config: Optional[Config] = None,
                 lib: Optional[str] = None):
        self._config = config or Config()
        self._m, self._lib = None, None
        if not Path(model_path).is_file():
            raise ValueError(f"Model path '{model_path}' doesn't exist.")
        if not model_type:
            if not is_gguf(model_path):
                raise ValueError("Unable to detect model type. Please specify a model type.")
            model_type = "gguf"
        self._lib = load_library(lib)
        self._m = self._lib.ctb_multi_create(model_path.encode(), model_type.encode(), self._config.to_struct(), n_slots)
        if self._m is None:
            raise RuntimeError(f"Failed to create a {n_slots}-slot MultiLLM from '{model_path}'.")
        info = (c_int * 6)()
        self._lib.ctb_multi_info(self._m, info)
        self.n_slots, self.vocab_size, self.n_embd, self.context_length, self.eos_token_id, self.bos_token_id = list(info)
        self._context: List[List[int]] = [[] for _ in range(self.n_slots)]

    config = property(lambda self: self._config)

    def context(self, slot: int) -> List[int]:
        """The tokens slot `slot` has evaluated since it was created or reset (LLM._context of that slot)."""
        return self._context[self._slot(slot)]

    def _slot(self, slot: int) -> int:
        if not 0 <= slot < self.n_slots:
            raise IndexError(f"slot {slot} is out of range (0 .. {self.n_slots - 1})")
        return slot

    def eval(self, tokens_by_slot: Dict[int, Sequence[int]], *, batch_size: Optional[int] = None, logits_all: bool = False) -> None:
        """Each listed slot evaluates its tokens after its own history (n_past = its context length), chunked by batch_size as
        LLM.eval chunks; all of them share batched launches.  logits_all=True also keeps the logits of every evaluated token:
        `all_logits` is then {slot: (n, vocab_size) float32 array}, each row what LLM.eval(..., logits_all=True) gives."""
        self.all_logits = None
        if not logits_all:
            self._eval_call(tokens_by_slot, batch_size, self._lib.ctb_multi_eval, ok=True)
            return
        import numpy as np
        slots = [self._slot(s) for s in tokens_by_slot]
        tokens_by_slot = {s: _check_ids(tokens_by_slot[s], self.vocab_size, f"slot {s}: token") for s in slots}
        rows = np.empty((sum(map(len, tokens_by_slot.values())), self.vocab_size), np.float32)
        self._eval_call(tokens_by_slot, batch_size, self._lib.ctb_multi_eval_rows, rows.ctypes.data_as(POINTER(c_float)))
        self.all_logits, at = {}, 0
        for s in slots:
            self.all_logits[s], at = rows[at:at + len(tokens_by_slot[s])], at + len(tokens_by_slot[s])

    def _eval_call(self, tokens_by_slot, batch_size, fn, *out, ok=0) -> None:
        """One ctb_multi_eval / ctb_multi_eval_rows / ctb_multi_eval_scored call, which returns `ok` on success: the slots'
        lists concatenated in dict order, each after its slot's context."""
        bs = _pick(batch_size, self._config.batch_size)
        slots = [self._slot(s) for s in tokens_by_slot]
        off, flat = _flatten([tokens_by_slot[s] for s in slots])
        n = len(slots)
        past = [len(self._context[s]) for s in slots]
        if fn(self._m, n, _ints(slots), _ints(off), _ints(flat), _ints(past), bs, *out) != ok:
            raise RuntimeError("Failed to evaluate tokens.")
        for s in slots:
            self._context[s].extend(tokens_by_slot[s])

    def score_many(self, requests: Sequence[Tuple[Sequence[int], Sequence[int]]], *, batch_size: Optional[int] = None) -> List[Tuple[float, bool]]:
        """The loglikelihood requests of an evaluation harness: for each (context_tokens, continuation_tokens), the sum of the
        continuation tokens' log-probabilities, each under the logits after the tokens before it, and whether every continuation
        token is the greedy pick there (LLM.score defines both).  Each request runs in a fresh slot; up to n_slots requests are
        admitted at once and share every launch.  The context must hold at least one token (BOS, say)."""
        import numpy as np
        reqs = []
        for i, (ctx, cont) in enumerate(requests):
            ctx, cont = _check_ids(ctx, self.vocab_size, f"request {i}: context token"), _check_ids(cont, self.vocab_size, f"request {i}: continuation token")
            if not ctx or not cont:
                raise ValueError(f"request {i}: the context and the continuation must each hold at least one token")
            if len(ctx) + len(cont) - 1 > self.context_length:
                raise ValueError(f"request {i}: {len(ctx) + len(cont) - 1} tokens to evaluate; the context length is {self.context_length}")
            reqs.append((ctx, cont))
        results: List[Tuple[float, bool]] = []
        for first in range(0, len(reqs), self.n_slots):
            group = reqs[first:first + self.n_slots]
            by_slot, targets = {}, []
            for s, (ctx, cont) in enumerate(group):
                self.reset(s)
                whole = ctx + cont
                by_slot[s] = whole[:-1]   # the last token's row scores nothing
                targets += [-1] * (len(ctx) - 1) + cont
            lp, gr = np.zeros(len(targets), np.float64), np.zeros(len(targets), np.int32)
            self._eval_call(by_slot, batch_size, self._lib.ctb_multi_eval_scored, _ints(targets), lp.ctypes.data_as(POINTER(c_double)),
                            gr.ctypes.data_as(POINTER(c_int)))
            at = 0
            for s, (ctx, cont) in enumerate(group):
                n = len(ctx) + len(cont) - 1
                mine, pick = lp[at + len(ctx) - 1:at + n], gr[at + len(ctx) - 1:at + n]
                results.append((float(np.sum(mine)), bool(np.all(pick != 0))))
                at += n
        return results

    def logits(self, slot: int) -> List[float]:
        p = self._lib.ctb_multi_logits(self._m, self._slot(slot))
        return Vector(p, self.vocab_size if p else 0)

    def embeddings(self, slot: int) -> List[float]:
        p = self._lib.ctb_multi_embeddings(self._m, self._slot(slot))
        return Vector(p, self.n_embd if p else 0)

    def greedy(self, slots: Sequence[int]) -> List[int]:
        """The greedy picks of these slots (what sample(top_k=1, repetition_penalty=1.0) returns), computed on the device."""
        slots = [self._slot(s) for s in slots]
        out = (c_int * max(len(slots), 1))()
        if self._lib.ctb_multi_greedy(self._m, len(slots), (c_int * max(len(slots), 1))(*slots), out) != 0:
            raise RuntimeError("No logits to pick from: every slot must have been evaluated.")
        return list(out[: len(slots)])

    def sample(self, slot: int, *, top_k=None, top_p=None, temperature=None, repetition_penalty=None, last_n_tokens=None, seed=None) -> int:
        """LLM.sample on this slot: the same defaults, its own last_n_tokens window."""
        return self.sample_many([slot], top_k=top_k, top_p=top_p, temperature=temperature, repetition_penalty=repetition_penalty,
                                last_n_tokens=last_n_tokens, seed=seed)[0]

    def sample_many(self, slots: Sequence[int], *, top_k=None, top_p=None, temperature=None, repetition_penalty=None, last_n_tokens=None,
                    seed=None) -> List[int]:
        """sample() of every listed slot, in one call: draw i is what LLM.sample returns with the i-th settings on an LLM fed
        slot slots[i]'s history.  Each setting is one value for every slot or a sequence with one value per slot (None: the
        config's).  The penalty and top-k cut of all slots run in one device launch; the host finishes each draw."""
        slots = [self._slot(s) for s in slots]
        n, cfg = len(slots), self._config
        args = {}
        for name, value in (("top_k", top_k), ("top_p", top_p), ("temperature", temperature), ("repetition_penalty", repetition_penalty),
                            ("last_n_tokens", last_n_tokens), ("seed", seed)):
            args[name] = [_pick(v, getattr(cfg, name)) for v in per_slot(value, n, name)]
        windows = [self._context[s][-(last_n if last_n >= 0 else self.context_length):]   # (last_n 0: the whole context, as LLM.sample)
                   for s, last_n in zip(slots, args["last_n_tokens"])]
        off, flat = _flatten(windows)
        out = (c_int * max(n, 1))()
        floats = lambda v: (c_float * max(n, 1))(*v)
        if self._lib.ctb_multi_sample_many(self._m, n, _ints(slots), _ints(off), _ints(flat), _ints(args["top_k"]), floats(args["top_p"]),
                                           floats(args["temperature"]), floats(args["repetition_penalty"]), _ints(args["seed"]), out) != 0:
            raise RuntimeError(f"Failed to sample slots {slots}: each must have logits and be listed once.")
        return list(out[:n])

    def device_samples(self) -> int:
        """Draws so far that the device answered (the rest ran the host sampler on a slot's logits)."""
        return self._lib.ctb_multi_device_samples(self._m)

    def reset(self, slot: int) -> None:
        """The slot starts over, as a fresh LLM."""
        self._lib.ctb_multi_reset(self._m, self._slot(slot))
        self._context[slot] = []

    def launches(self) -> int:
        return self._lib.ctb_multi_launches(self._m)

    def last_eval_ms(self) -> float:
        return self._lib.ctb_multi_last_eval_ms(self._m)

    def fork(self, src: int, dsts: Sequence[int]) -> None:
        """Each slot in dsts becomes a copy of slot src, device to device: its KV cache, last results and tokens."""
        src, dsts = self._slot(src), [self._slot(d) for d in dsts]
        if src in dsts:
            raise ValueError(f"slot {src} cannot be forked into itself")
        if self._lib.ctb_multi_fork(self._m, src, len(dsts), (c_int * max(len(dsts), 1))(*dsts)) != 0:
            raise RuntimeError(f"Failed to fork slot {src}.")
        for d in dsts:
            self._context[d] = list(self._context[src])

    def save(self, slot: int) -> SequenceState:
        """What slot `slot` has evaluated, for restore into any slot here, another MultiLLM or an LLM of the same model file."""
        slot = self._slot(slot)
        return state.save(partial(self._lib.ctb_multi_state_size, self._m), partial(self._lib.ctb_multi_save, self._m, slot),
                          self._context[slot])

    def restore(self, slot: int, saved: SequenceState) -> None:
        """The slot continues from a saved state exactly as if it had just evaluated the state's tokens."""
        slot = self._slot(slot)
        self._context[slot] = state.restore(self._lib, saved, partial(self._lib.ctb_multi_restore, self._m, slot))

    def generate_many(self, prompts: Sequence[Sequence[int]], max_new_tokens: int, *, n: int = 1, seeds: Optional[Sequence[int]] = None,
                      batch_size: Optional[int] = None, **sampling) -> list:
        """Generates for every prompt, up to n_slots at once: a sequence ends at EOS (not included) or after max_new_tokens, and
        its slot takes the next waiting prompt, whose prompt tokens then share launches with the other slots' decode tokens.
        Each result equals LLM.generate of that prompt on a fresh LLM with the same sampling arguments.

        n > 1 draws n samples of every prompt: the prompt is evaluated once, in one slot, which is then forked into n - 1 more;
        sample j draws with seed seeds[j] (required: equal seeds draw equal samples).  The result of a prompt is then the list
        of its n samples, sample j equal to LLM.generate(prompt, seed=seeds[j], ...) on a fresh LLM."""
        if not 1 <= n <= self.n_slots:
            raise ValueError(f"n = {n}: each prompt's samples need a slot each, and there are {self.n_slots}")
        if (n > 1 or seeds is not None) and (seeds is None or len(seeds) != n):
            raise ValueError(f"n = {n} samples per prompt need n seeds (equal seeds draw equal samples)")
        results: List[List[Optional[List[int]]]] = [[None] * n for _ in prompts]
        waiting = list(range(len(prompts)))[::-1]
        owner: Dict[int, Tuple[int, int]] = {}   # slot -> (prompt index, sample index)
        pending: Dict[int, List[int]] = {}
        forks: Dict[int, List[int]] = {}          # slot evaluating a prompt -> the slots it is forked into after that eval
        free = list(range(self.n_slots))

        def admit():
            while waiting and len(free) >= n:
                i, group = waiting.pop(), free[:n]
                del free[:n]
                self.reset(group[0])
                pending[group[0]], forks[group[0]] = list(prompts[i]), group[1:]
                for j, s in enumerate(group):
                    owner[s], results[i][j] = (i, j), []

        admit()
        while owner:
            self.eval(pending, batch_size=batch_size)
            pending = {}
            for s, dsts in forks.items():
                if dsts:
                    self.fork(s, dsts)
            forks = {}
            order = sorted(owner)
            kw = sampling if seeds is None else {**sampling, "seed": [seeds[owner[s][1]] for s in order]}
            for slot, tok in zip(order, self.sample_many(order, **kw)):
                i, j = owner[slot]
                if tok == self.eos_token_id or max_new_tokens <= 0:
                    done = True
                else:
                    results[i][j].append(tok)
                    done = len(results[i][j]) >= max_new_tokens
                    pending[slot] = [tok]
                if done:
                    pending.pop(slot, None)
                    del owner[slot]
                    free.append(slot)
                    admit()
        return results if n > 1 else [r[0] for r in results]

    def beam_search(self, prompt_tokens: Sequence[int], n_beams: int, max_new_tokens: int, *, batch_size: Optional[int] = None) -> Tuple[List[int], float]:
        """Beam search after the prompt, as the reference's llama_beam_search with its example's callback (a beam ends at EOS):
        (the winning beam's tokens, an EOS included when it ends in one; its p, renormalised over the last step's beams), bit
        for bit.  The prompt is evaluated in one slot, chunked by batch_size; the search holds n_beams slots and evaluates all
        live beams in one batched launch per step.  It uses the lowest n_beams slots and resets them afterwards: their earlier
        context is not kept."""
        return self.beam_search_many([prompt_tokens], n_beams, max_new_tokens, batch_size=batch_size)[0]

    def beam_search_many(self, prompts: Sequence[Sequence[int]], n_beams: int, max_new_tokens: int, *,
                         batch_size: Optional[int] = None) -> List[Tuple[List[int], float]]:
        """beam_search of every prompt: up to n_slots // n_beams searches at once, a prompt admitted as slots free up, the live
        beams of all of them evaluated in the same launches.  Each result equals beam_search of that prompt alone.  The slots
        used, the lowest n_beams * min(len(prompts), n_slots // n_beams), are reset afterwards."""
        if not 1 <= n_beams <= min(self.n_slots, self.vocab_size):
            raise ValueError(f"n_beams = {n_beams}: each beam needs a slot, and there are {self.n_slots}")
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must not be negative")
        prompts = [_check_ids(p, self.vocab_size, f"prompt {i}: token") for i, p in enumerate(prompts)]
        for i, p in enumerate(prompts):
            if not p:
                raise ValueError(f"prompt {i} is empty")
            if len(p) + max_new_tokens > self.context_length:
                raise ValueError(f"prompt {i}: {len(p)} tokens and {max_new_tokens} more exceed the context length {self.context_length}")
        off, flat = _flatten(prompts)
        n = len(prompts)
        out_off = (c_int * (n + 1))()
        out_tok = (c_int * max(n * max_new_tokens, 1))()
        out_p = (c_float * max(n, 1))()
        rc = self._lib.ctb_multi_beam_search(self._m, n, _ints(off), _ints(flat), n_beams, max_new_tokens, _pick(batch_size, self._config.batch_size),
                                             out_off, out_tok, out_p)
        # searches take the lowest free slots, n_beams each: these are the slots used, and the library has reset them
        for s in range(n_beams * min(n, self.n_slots // n_beams) if max_new_tokens > 0 else 0):
            self._context[s] = []
        if rc != 0:
            raise RuntimeError(f"Beam search failed (n_beams = {n_beams}); see stderr.")
        return [(list(out_tok[out_off[i]:out_off[i + 1]]), float(out_p[i])) for i in range(n)]

    def beam_stats(self) -> Dict[str, float]:
        """The last beam search: steps, host-clock ms of its evals, of its row fetches + selections and of its re-parentings,
        the K / V bytes the re-parenting launches moved, the tokens evaluated (prompts included), the steps that also evaluated
        a prompt and the ms of their evals."""
        v = (c_double * 8)()
        self._lib.ctb_multi_beam_stats(self._m, v)
        return dict(zip(("steps", "eval_ms", "select_ms", "reparent_ms", "reparent_bytes", "tokens", "prompt_steps", "prompt_eval_ms"), list(v)))

    def __del__(self):
        if self.__dict__.get("_m") is not None and self.__dict__.get("_lib") is not None:
            self._lib.ctb_multi_delete(self._m)
            self._m = None
