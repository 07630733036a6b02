"""The grammars the grammar tests run (written for this project).  GRAMMARS: name -> GBNF text the reference parser accepts.
REFUSED: name -> (text, words the refusal's message holds)."""
from pathlib import Path

import numpy as np

from ctransformers_b200 import synth

JSON = r'''
root   ::= object
value  ::= object | array | string | number | ("true" | "false" | "null") ws

object ::=
  "{" ws (
            string ":" ws value
    ("," ws string ":" ws value)*
  )? "}" ws

array  ::=
  "[" ws (
            value
    ("," ws value)*
  )? "]" ws

string ::=
  "\"" (
    [^"\\] |
    "\\" (["\\/bfnrt] | "u" [0-9a-fA-F] [0-9a-fA-F] [0-9a-fA-F] [0-9a-fA-F])
  )* "\"" ws

number ::= ("-"? ([0-9] | [1-9] [0-9]*)) ("." [0-9]+)? ([eE] [-+]? [0-9]+)? ws

ws ::= ([ \t\n] ws)?
'''

ARITHMETIC = r'''
root  ::= (expr "=" ws term "\n")+
expr  ::= term ([-+*/] term)*
term  ::= ident | num | "(" ws expr ")" ws
ident ::= [a-z] [a-z0-9_]* ws
num   ::= [0-9]+ ws
ws    ::= [ \t\n]*
'''

LIST = r'''
root ::= item+
# an item: a dash, a space, then words
item ::= "- " [^\r\n\x0b\x0c\x85\u2028\u2029]+ "\n"
'''

NON_ASCII = r'''
root   ::= (word " ")* word "。"?
word   ::= latin | cjk | other
latin  ::= [a-zA-Zàâçéèêëîïôûùüÿñæœ]+
cjk    ::= [一-鿿ぁ-ゟ゠-ヿ]+
other  ::= [^\x00-\x7F] [^\x00-\x7F]?
'''

OPERATORS = r'''
root ::= a? (b | c)* d+ e ("x" | ) ( ( "y" | "z" )* "w" )? tail
a    ::= "a" | "\x41" # a or A
b    ::= "b\n" | "\u00e9"
c    ::= [c-e] | "\U0001F600"
d    ::= "d"
e    ::= ( )  "e" | "E"
tail ::= "\t" | "\r" | [\[\]\\"] |
'''

FIXED = r'''
root ::= "ok"
'''

NOTHING = r'''
root ::= [\x00]
'''


def deep_chain(n: int = 300) -> str:
    """root ::= "t" r1;  r_i ::= r_{i+1} "a";  r_n ::= "h" "a": for a piece like "th" a thread must expand n references at once
    after the "t", and every expansion keeps the "a" after it on the stack, which no small per-thread pool holds."""
    lines = ['root ::= "t" r1 | "y"']
    for i in range(1, n):
        lines.append(f'r{i} ::= r{i + 1} "a"')
    lines.append(f'r{n} ::= "h" "a"')
    return "\n".join(lines) + "\n"


DEEP = deep_chain()

GRAMMARS = {"json": JSON, "arithmetic": ARITHMETIC, "list": LIST, "non_ascii": NON_ASCII, "operators": OPERATORS,
            "fixed": FIXED, "nothing": NOTHING, "deep": DEEP}

REFUSED = {
    "syntax_missing_assign": ("root \"x\"\n", "expecting ::="),
    "syntax_unclosed_group": ("root ::= ( \"x\" \n", "expecting ')'"),
    "syntax_bad_escape": ("root ::= \"\\q\"\n", "unknown escape"),
    "syntax_short_hex": ("root ::= \"\\x4\"\n", "expecting 2 hex chars"),
    "syntax_dangling_star": ("root ::= * \"x\"\n", "expecting preceeding item"),
    "syntax_unterminated": ("root ::= \"abc", "unexpected end of input"),
    "no_root": ("start ::= \"x\"\n", "'root'"),
    "undefined": ("root ::= a b\na ::= \"x\"\n", "undefined rule 'b'"),
    "left_recursion": ("root ::= expr\nexpr ::= expr \"+\" num | num\nnum ::= [0-9]\n", "left recursion"),
    "left_recursion_nullable": ("root ::= a\na ::= b a \"x\" | \"y\"\nb ::= \"z\" |\n", "left recursion"),
}


# ---- the golden runs (make_golden_grammar.py): models, grammars and sampler settings
# name: (arch, shape, ftype, ctx, extra_pieces).  The mask depends only on the vocabulary, so the 32000 / 65024 entries ride on
# tiny widths.
MODELS = {
    "llama_tiny_q4km": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=3, n_ctx_train=256), "Q4_K_M", 96, False),
    "falcon_tiny_q5km": ("falcon", synth.FalconShape(n_vocab=1024, n_embd=512, n_head=8, n_head_kv=1, n_ff=2048, n_layer=2, n_ctx_train=256), "Q5_K_M", 96, False),
    "llama_gqa_q5km": ("llama", synth.LlamaShape(n_vocab=2048, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2816, n_layer=2, n_ctx_train=256), "Q5_K_M", 96, False),
    "llama_extra_q4km": ("llama", synth.LlamaShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=2, n_ctx_train=256), "Q4_K_M", 96, True),
    "falcon_extra_q5km": ("falcon", synth.FalconShape(n_vocab=1024, n_embd=256, n_head=4, n_head_kv=1, n_ff=1024, n_layer=2, n_ctx_train=256), "Q5_K_M", 96, True),
    "llama_v32000": ("llama", synth.LlamaShape(n_vocab=32000, n_embd=256, n_head=4, n_head_kv=4, n_ff=768, n_layer=1, n_ctx_train=256), "Q4_K_M", 96, True),
    "falcon_v65024": ("falcon", synth.FalconShape(n_vocab=65024, n_embd=256, n_head=4, n_head_kv=1, n_ff=1024, n_layer=1, n_ctx_train=256), "Q5_K_M", 96, True),
}
PROMPT_LEN, MAX_NEW = 12, 16
# name: (top_k, top_p, temperature, repetition_penalty, last_n_tokens, seed)
SETTINGS = {"greedy": (1, 1.0, 1.0, 1.0, 64, 0), "default": (40, 0.95, 0.8, 1.1, 64, 7)}
RUN_GRAMMARS = ["json", "arithmetic", "fixed", "non_ascii", "list"]


def build_model(name, directory):
    arch, shape, ftype, ctx, extra = MODELS[name]
    path = Path(directory) / f"grammar_{name}.gguf"
    if not path.exists():
        (synth.write_llama if arch == "llama" else synth.write_falcon)(path, shape, ftype, seed=11, extra_pieces=extra)
    return path, ctx


def prompt(name):
    arch, shape, _, _, _ = MODELS[name]
    ids = np.random.default_rng(3).integers(259 if arch == "llama" else 300, min(shape.n_vocab, 1000), PROMPT_LEN).tolist()
    if arch == "llama":
        ids[0] = 1
    return ids


def runs():
    """key -> (model, grammar, settings)"""
    return {f"{m}__{g}__{s}": (m, g, s) for m in MODELS for g in RUN_GRAMMARS for s in SETTINGS}


def pieces_of(path):
    """Every token's piece (llama_token_to_str) of a model file, through the library's host-only vocabulary."""
    import ctypes as C
    from ctransformers_b200.lib import load_library
    lib = load_library()
    v = lib.ctb_vocab_load(str(path).encode())
    buf, out = C.create_string_buffer(1024), []
    for t in range(lib.ctb_vocab_size(v)):
        n = lib.ctb_vocab_piece(v, t, buf, len(buf))
        out.append(buf.raw[:n])
    lib.ctb_vocab_free(v)
    return out
