"""Sequence states, host side: ctb_state_info parses and checks a blob's header without a device, and SequenceState survives a
pickle round trip (include/ctransformers_b200.h ctb_state_header)."""
import ctypes as C
import pickle
import struct

import numpy as np
import pytest

MAGIC, VERSION = 0x53425443, 1
HEADER = "<IIiiiiiiiiQ"   # magic, version, n_layer, n_head_kv, head_dim, k_stride, n_embd, n_vocab, n_tokens, has_results, fingerprint


def blob(n_tokens=5, n_layer=2, n_kv=2, hd=80, ks=80, n_embd=640, n_vocab=100, results=1, magic=MAGIC, version=VERSION, fp=0x1234):
    rng = np.random.default_rng(n_tokens)
    head = struct.pack(HEADER, magic, version, n_layer, n_kv, hd, ks, n_embd, n_vocab, n_tokens, results, fp)
    toks = rng.integers(0, n_vocab, n_tokens).astype("<i4").tobytes()
    n_pad = -(-n_tokens // 256) * 256                     # V rows hold whole 256-position blocks
    kv = rng.integers(0, 1 << 16, n_layer * n_kv * (n_tokens * ks + n_pad * hd)).astype("<u2").tobytes()
    res = rng.standard_normal(n_vocab + n_embd).astype("<f4").tobytes() if results else b""
    return head + toks + kv + res


def info(lib, data):
    from ctransformers_b200.lib import StateHeader
    h = StateHeader()
    rc = lib.ctb_state_info(data, len(data), C.byref(h))
    return rc, h


def test_header_layout():
    from ctransformers_b200.lib import StateHeader
    assert C.sizeof(StateHeader) == struct.calcsize(HEADER) == 48


@pytest.mark.parametrize("n_tokens,results", [(0, 0), (1, 1), (37, 1), (37, 0), (256, 1), (300, 1)])
def test_state_info_accepts_a_hand_built_header(lib, n_tokens, results):
    data = blob(n_tokens=n_tokens, results=results, ks=88, hd=84)
    rc, h = info(lib, data)
    assert rc == 0
    assert (h.magic, h.version, h.n_layer, h.n_head_kv, h.head_dim, h.k_stride, h.n_embd, h.n_vocab, h.n_tokens, h.has_results,
            h.fingerprint) == (MAGIC, VERSION, 2, 2, 84, 88, 640, 100, n_tokens, results, 0x1234)


def test_state_info_refusals(lib, capfd):
    good = blob()
    cases = {
        "bad magic": (blob(magic=0x12345678), "bad magic"),
        "bad version": (blob(version=2), "version 2"),
        "truncated": (good[:-1], "disagrees with its header"),
        "one byte too many": (good + b"\0", "disagrees with its header"),
        "shorter than a header": (good[:20], "header"),
        "token count against size": (bytearray(good[:32]) + struct.pack("<i", 6) + good[36:], "disagrees with its header"),
        "k_stride below head_dim": (blob(ks=64, hd=80), "malformed"),
        "negative token count": (bytearray(good[:32]) + struct.pack("<i", -1) + good[36:], "malformed"),
    }
    for what, (data, msg) in cases.items():
        rc, _ = info(lib, bytes(data))
        assert rc == -1, what
        assert msg in capfd.readouterr().err, what


def test_sequence_state_pickles():
    from ctransformers_b200 import SequenceState
    s = SequenceState([1, 5, 9], bytearray(blob(n_tokens=3)))
    t = pickle.loads(pickle.dumps(s))
    assert t.tokens == [1, 5, 9] and t.n_past == 3 and t.data == s.data


def test_restore_checks_the_tokens_against_the_blob(lib):
    """The Python side refuses a SequenceState whose tokens are not the blob's before any library call touches a handle."""
    from ctransformers_b200 import SequenceState
    from ctransformers_b200.state import restore
    data = blob(n_tokens=4)
    held = np.frombuffer(data[48:64], "<i4").tolist()
    calls = []
    load = lambda buf, size: calls.append(size) or 0
    assert restore(lib, SequenceState(held, data), load) == held and calls == [len(data)]
    with pytest.raises(ValueError):
        restore(lib, SequenceState(held[:3] + [held[3] + 1], data), load)
    with pytest.raises(ValueError):
        restore(lib, SequenceState(held, data[:-2]), load)
    assert calls == [len(data)]
