"""Writes the grammar goldens from the UNMODIFIED reference:  python tests/golden/make_golden_grammar.py

Needs the reference sources (REF, default /root/reference): the reference's own grammar_parser::parse is compiled together with
tests/grammar_parser_shim.cpp into a temporary library, and the sampler chain runs through oracle/_ref/libctransformers_ref.so
(built by oracle/Makefile), which exports llama_grammar_* and llama_sample_*.

  grammar_rules.npz  for every grammar of tests/grammar_cases.py GRAMMARS:
    <name>_off, <name>_elems   the parsed rules: rule r is elems[off[r] .. off[r + 1]) of (type, value) rows
    <name>_sym_names, <name>_sym_ids   parse_state.symbol_ids
  and for every REFUSED case, refused_<name>: whether the reference parser refused the text itself (it returns an empty state).

  grammar_runs.npz  for every run of grammar_cases.runs() (model, grammar, settings): the prompt is evaluated through llama.cpp's
  C API in chunks of 8 (LLM.generate's eval), then each step reseeds (llama_set_rng_seed), applies llama_sample_repetition_penalty
  over the last 64 tokens of the context, llama_sample_grammar, top-k, top-p, temperature, llama_sample_token (ctransformers'
  Sample, models/llms/llama.cc:53-84, with the grammar where examples/main/main.cpp:650-695 puts it), then
  llama_grammar_accept_token and the eval of the token, until EOS, MAX_NEW tokens or a token the accept aborts on.
    <key>_tokens   the drawn tokens (EOS included when drawn)
    <key>_allowed  per step, the tokens llama_sample_grammar leaves finite, packed with np.packbits
    <key>_dead_end the run ended on a drawn token that llama_grammar_accept_token aborts on (the mask allows a piece with an
                   overlong-encoded NUL, the accept cannot take the NUL); it is the last of the tokens
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import grammar_cases as G  # noqa: E402
from make_golden_logits_all import RefContext, reference  # noqa: E402

REF = Path(os.environ.get("REF", "/root/reference"))


class Elem(C.Structure):
    _fields_ = [("type", C.c_int), ("value", C.c_uint32)]   # llama_grammar_element, llama.h:197-200


class TokenData(C.Structure):
    _fields_ = [("id", C.c_int), ("logit", C.c_float), ("p", C.c_float)]   # llama_token_data


class TokenDataArray(C.Structure):
    _fields_ = [("data", C.POINTER(TokenData)), ("size", C.c_size_t), ("sorted", C.c_bool)]


def parser(tmp):
    llama = REF / "models" / "submodules" / "llama.cpp"
    so = Path(tmp) / "libgrammar_ref.so"
    subprocess.check_call(["g++", "-std=c++11", "-O2", "-fPIC", "-shared", "-w", f"-I{llama}", f"-I{llama / 'common'}",
                           str(HERE.parent / "grammar_parser_shim.cpp"), str(llama / "common" / "grammar-parser.cpp"), "-o", str(so)])
    p = C.CDLL(str(so))
    p.gp_parse.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    p.gp_rules.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_uint)]
    p.gp_symbol.argtypes = [C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_uint)]
    return p


def parse(p, text):
    """(off, elems (n, 2), names, ids) of the reference parser, or None when it refuses the text."""
    nr, ne, ns = C.c_int(), C.c_int(), C.c_int()
    if p.gp_parse(text.encode(), C.byref(nr), C.byref(ne), C.byref(ns)) != 0:
        return None
    off, el = (C.c_int * (nr.value + 1))(), (C.c_uint * (2 * ne.value))()
    p.gp_rules(off, el)
    names, ids, buf, rid = [], [], C.create_string_buffer(4096), C.c_uint()
    for i in range(ns.value):
        n = p.gp_symbol(i, buf, len(buf), C.byref(rid))
        names.append(buf.raw[:n].decode())
        ids.append(rid.value)
    return np.array(off[:], np.int32), np.array(el[:], np.uint32).reshape(-1, 2), names, ids


def ref_grammar(r, off, elems):
    """llama_grammar_init over the parsed rules at `root`"""
    arrays = [(Elem * (off[i + 1] - off[i]))(*[Elem(int(t), int(v)) for t, v in elems[off[i]:off[i + 1]]]) for i in range(len(off) - 1)]
    ptrs = (C.POINTER(Elem) * len(arrays))(*[C.cast(a, C.POINTER(Elem)) for a in arrays])
    return arrays, ptrs


def accepts(r, ctx, gram, tok):
    """Whether llama_grammar_accept_token takes tok without aborting, tried in a forked child.  It aborts where no stack is
    left, which happens after the mask allowed a piece holding an overlong-encoded NUL: the mask ends such a piece at the NUL,
    accept feeds the NUL to the stacks."""
    pid = os.fork()
    if pid == 0:
        os.close(2)   # the abort's message
        r.llama_grammar_accept_token(ctx, gram, tok)
        os._exit(0)
    _, status = os.waitpid(pid, 0)
    return os.WIFEXITED(status) and os.WEXITSTATUS(status) == 0


def main():
    r = reference()
    r.llama_grammar_init.restype = C.c_void_p
    r.llama_grammar_init.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t]
    r.llama_grammar_free.argtypes = [C.c_void_p]
    r.llama_grammar_accept_token.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    r.llama_sample_grammar.argtypes = [C.c_void_p, C.POINTER(TokenDataArray), C.c_void_p]
    r.llama_sample_repetition_penalty.argtypes = [C.c_void_p, C.POINTER(TokenDataArray), C.POINTER(C.c_int), C.c_size_t, C.c_float]
    r.llama_sample_top_k.argtypes = [C.c_void_p, C.POINTER(TokenDataArray), C.c_int, C.c_size_t]
    r.llama_sample_top_p.argtypes = [C.c_void_p, C.POINTER(TokenDataArray), C.c_float, C.c_size_t]
    r.llama_sample_temperature.argtypes = [C.c_void_p, C.POINTER(TokenDataArray), C.c_float]
    r.llama_sample_token.argtypes = [C.c_void_p, C.POINTER(TokenDataArray)]
    r.llama_sample_token.restype = C.c_int
    r.llama_set_rng_seed.argtypes = [C.c_void_p, C.c_uint32]
    r.llama_token_eos.argtypes = [C.c_void_p]
    r.llama_token_eos.restype = C.c_int
    rules, runs = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        p = parser(tmp)
        parsed = {}
        for name, text in G.GRAMMARS.items():
            got = parse(p, text)
            assert got is not None, name
            parsed[name] = got
            off, el, names, ids = got
            rules[f"{name}_off"], rules[f"{name}_elems"] = off, el
            rules[f"{name}_sym_names"], rules[f"{name}_sym_ids"] = np.array(names), np.array(ids, np.int32)
        for name, (text, _) in G.REFUSED.items():
            rules[f"refused_{name}"] = np.array(parse(p, text) is None)
        np.savez_compressed(HERE / "grammar_rules.npz", **rules)
        for model in G.MODELS:
            path, ctx = G.build_model(model, tmp)
            n_vocab = G.MODELS[model][1].n_vocab
            for gname in G.RUN_GRAMMARS:
                off, el, _, _ = parsed[gname]
                root = dict(zip(parsed[gname][2], parsed[gname][3]))["root"]
                for sname, (top_k, top_p, temp, pen, last_n, seed) in G.SETTINGS.items():
                    key = f"{model}__{gname}__{sname}"
                    ref = RefContext(r, path, ctx, n_vocab)
                    eos = r.llama_token_eos(ref.ctx)
                    arrays, ptrs = ref_grammar(r, off, el)
                    gram = r.llama_grammar_init(ptrs, len(arrays), root)
                    context = G.prompt(model)
                    blocks = ref.batch_eval(context, 8)
                    last = blocks[-1][-1]
                    tokens, allowed, dead_end = [], [], False
                    for _ in range(G.MAX_NEW):
                        # the bitmap: llama_sample_grammar over zeros
                        z = (TokenData * n_vocab)(*[TokenData(i, 0.0, 0.0) for i in range(n_vocab)])
                        za = TokenDataArray(z, n_vocab, False)
                        r.llama_sample_grammar(ref.ctx, C.byref(za), gram)
                        allowed.append(np.packbits(np.isfinite(np.array([z[i].logit for i in range(n_vocab)]))))
                        cand = (TokenData * n_vocab)(*[TokenData(i, float(last[i]), 0.0) for i in range(n_vocab)])
                        arr = TokenDataArray(cand, n_vocab, False)
                        window = context[-last_n:]
                        win = (C.c_int * max(len(window), 1))(*window)
                        r.llama_set_rng_seed(ref.ctx, seed)
                        r.llama_sample_repetition_penalty(ref.ctx, C.byref(arr), win, len(window), pen)
                        r.llama_sample_grammar(ref.ctx, C.byref(arr), gram)
                        r.llama_sample_top_k(ref.ctx, C.byref(arr), top_k, 1)
                        r.llama_sample_top_p(ref.ctx, C.byref(arr), top_p, 1)
                        r.llama_sample_temperature(ref.ctx, C.byref(arr), temp)
                        tok = r.llama_sample_token(ref.ctx, C.byref(arr))
                        tokens.append(tok)
                        if not accepts(r, ref.ctx, gram, tok):
                            dead_end = True   # the mask allowed it, but the reference's accept aborts on it
                            break
                        r.llama_grammar_accept_token(ref.ctx, gram, tok)
                        if tok == eos:
                            break
                        context.append(tok)
                        last = ref.batch_eval([tok], 8)[-1][-1]
                    r.llama_grammar_free(gram)
                    ref.close()
                    runs[f"{key}_tokens"] = np.array(tokens, np.int32)
                    runs[f"{key}_allowed"] = np.stack(allowed)
                    runs[f"{key}_dead_end"] = np.array(dead_end)
                    print(key, tokens, flush=True)
    np.savez_compressed(HERE / "grammar_runs.npz", **runs)


if __name__ == "__main__":
    main()
