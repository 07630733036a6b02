"""Grammar-constrained sampling on the host (csrc/grammar.hpp): the parser against the reference's grammar_parser::parse, the
refusals, the accept / mask of every golden run, and the UTF-8 and EOS rules of llama_sample_grammar, checked directly."""
from pathlib import Path

import numpy as np
import pytest

import grammar_cases as G
from ctransformers_b200 import Grammar

GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def rules():
    return np.load(GOLDEN / "grammar_rules.npz")


@pytest.fixture(scope="module")
def runs():
    return np.load(GOLDEN / "grammar_runs.npz")


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    d = tmp_path_factory.mktemp("grammar_models")
    return lambda name: G.build_model(name, d)[0]


@pytest.mark.parametrize("name", sorted(G.GRAMMARS))
def test_rules_and_symbols_equal_the_reference_parser(rules, name):
    g = Grammar(G.GRAMMARS[name])
    off, elems = rules[f"{name}_off"], rules[f"{name}_elems"]
    want = [[tuple(int(x) for x in e) for e in elems[off[r]:off[r + 1]]] for r in range(len(off) - 1)]
    assert g.rules == want
    assert g.symbol_ids == dict(zip(rules[f"{name}_sym_names"].tolist(), rules[f"{name}_sym_ids"].tolist()))


@pytest.mark.parametrize("name", sorted(G.REFUSED))
def test_refusals_raise_with_the_message(rules, name):
    text, words = G.REFUSED[name]
    with pytest.raises(ValueError, match="at byte") as e:
        Grammar(text)
    assert words in str(e.value)
    if name.startswith("syntax"):
        assert bool(rules[f"refused_{name}"])     # the reference parser refuses these too
    else:
        assert not bool(rules[f"refused_{name}"])  # it parses these, then fails (or recurses) where the rules are used


def eos_of(name):
    return 2 if G.MODELS[name][0] == "llama" else 11


@pytest.mark.parametrize("key", sorted(G.runs()))
def test_host_accept_and_mask_replay_every_golden_step(runs, models, key):
    model, gname, _ = G.runs()[key]
    pieces = G.pieces_of(models(model))
    eos = eos_of(model)
    state = Grammar(G.GRAMMARS[gname]).start()
    tokens, allowed = runs[f"{key}_tokens"], runs[f"{key}_allowed"]
    for step, tok in enumerate(tokens):
        mask = state.mask_pieces(pieces, eos)
        want = np.unpackbits(allowed[step])[:len(pieces)].astype(bool)
        assert np.array_equal(mask, want), (step, np.flatnonzero(mask != want)[:10])
        assert mask[tok]
        if bool(runs[f"{key}_dead_end"]) and step == len(tokens) - 1:
            # the mask allowed a piece with an overlong-encoded NUL that no stack takes: the reference aborts, this refuses
            with pytest.raises(ValueError):
                state.accept_piece(pieces[tok])
            break
        if tok == eos:
            assert state.allowed_eos
            break
        state.accept_piece(pieces[tok])


def test_fixed_string_leaves_only_eos():
    pieces = [b"", b"<s>", b"</s>", b"o", b"k", b"ok", b"okk", b"x"]
    s = Grammar(G.FIXED).start()
    assert not s.allowed_eos
    assert s.mask_pieces(pieces, 2).tolist() == [False, False, False, True, False, True, False, False]
    s.accept_piece(b"ok")
    assert s.allowed_eos
    assert s.mask_pieces(pieces, 2).tolist() == [False, False, True, False, False, False, False, False]
    with pytest.raises(ValueError):
        s.accept_piece(b"k")
    s.accept_piece(b"", eos=True)


def test_eos_needs_an_empty_stack():
    s = Grammar('root ::= "a" "b"?').start()
    with pytest.raises(ValueError):
        s.accept_piece(b"", eos=True)
    stacks_before = s.stacks
    with pytest.raises(ValueError):
        s.accept_piece(b"b")            # refused: the state stays as it was
    assert s.stacks == stacks_before
    s.accept_piece(b"a")
    assert s.allowed_eos                # "b"? can end here
    s.accept_piece(b"", eos=True)


def test_empty_and_nul_pieces_are_rejected():
    s = Grammar('root ::= [^x]*').start()
    pieces = [b"", b"\x00", b"\x00a", b"a\x00b", b"a", b"x"]
    # an empty piece or one starting with NUL is rejected; a NUL inside cuts the piece (the reference decodes a C string)
    assert s.mask_pieces(pieces, -1).tolist() == [False, False, False, True, True, False]


def test_partial_utf8_sequences():
    cjk = Grammar('root ::= [一-鿿]+').start()
    ri = "日".encode()   # e6 97 a5
    pieces = [ri[:1], ri[:2], ri, ri[1:], b"\xff", b"\xc3", b"a", "é".encode()[:1], "😀".encode()[:2]]
    # a lead byte whose completions can reach the range is allowed; a continuation first, 0xff, ASCII, a 2-byte lead are not;
    # a 4-byte lead's completions lie above the range
    assert cjk.mask_pieces(pieces, -1).tolist() == [True, True, True, False, False, False, False, False, False]
    cjk.accept_piece(ri[:1])
    _, partial = cjk.stacks
    assert partial == (ri[0] & 0x0F, 2)
    # now only continuation bytes fit, and only those that keep the code point in range
    after = [ri[1:2], ri[1:], b"a", ri, b"\xbf\xbf", b"\x80"]
    assert cjk.mask_pieces(after, -1).tolist() == [True, True, False, False, True, True]
    cjk.accept_piece(ri[1:])
    assert cjk.stacks[1] == (0x65E5, 0)
    low = Grammar('root ::= [一-鿿]').start()
    low.accept_piece(b"\xe4")   # completions 0x4000 .. 0x4fff: only continuations from 0xb8 on reach 0x4e00
    assert low.mask_pieces([b"\x80", b"\xb7", b"\xb8", b"\xbf"], -1).tolist() == [False, False, True, True]
    neg = Grammar('root ::= [^\\x00-\\x7F]').start()
    # an overlong 2-byte lead (0xc0, 0xc1) can complete to nothing valid
    assert neg.mask_pieces([b"\xc0", b"\xc2", b"\xe0", b"\xf0", b"A"], -1).tolist() == [False, True, True, True, False]


def test_invalid_sequences_are_rejected_everywhere():
    s = Grammar('root ::= [^a]* | "a"').start()
    # a continuation byte first is invalid; inside a new sequence the decoder does not check continuations (as the reference)
    assert s.mask_pieces([b"\x80", b"\xe6\x41", b"\xe6\x97\xa5", b"b"], -1).tolist() == [False, True, True, True]
    s.accept_piece(b"\xe6")
    # after a pending lead byte, a byte that is no continuation makes the sequence invalid
    assert s.mask_pieces([b"A", b"\x97\xa5", b"\x97"], -1).tolist() == [False, True, True]


def test_copy_is_independent():
    a = Grammar(G.ARITHMETIC).start()
    b = a.copy()
    a.accept_piece(b"x")
    assert a.stacks != b.stacks
    b.accept_piece(b"x")
    assert a.stacks == b.stacks


def test_an_overlong_nul_ends_the_candidate():
    # the reference ends a candidate's code points at the first 0, so an overlong-encoded NUL ends the piece for the mask
    s = Grammar('root ::= [a-z]+').start()
    pieces = [b"\xc0\x80", b"a\xe0\x80\x80b", b"\xe0\x80\x80b", b"1\xc0\x80", b"\xe0\x80", b"a\xc0\x80\xff"]
    assert s.mask_pieces(pieces, -1).tolist() == [True, True, True, False, False, False]
    # accepting the token feeds every code point, the 0 included: no stack takes it (the reference aborts there)
    with pytest.raises(ValueError):
        s.accept_piece(b"a\xe0\x80\x80b")
    # a pending sequence of value 0 completed by continuation bytes
    s.accept_piece(b"a")
    s.accept_piece(b"\xe0")
    assert s.stacks[1] == (0, 2)
    assert s.mask_pieces([b"\x80\x80", b"\x80", b"\x80\x80z"], -1).tolist() == [True, False, True]
