"""Multi-sequence decoding, host side: how ctb_multi_eval turns the slots' token lists into batched launches (ctb_multi_pack),
and the refusal without a GPU."""
import ctypes as C

import numpy as np
import pytest

PB_T = 32


def batch_eval_list(n_tokens, n_past, batch_size, n_ctx):
    """Positions and row lengths of LLM::BatchEval (llm.h:40-54): chunks of min(batch_size, n_ctx), n_past clamped per chunk."""
    bs = max(1, min(n_ctx, batch_size))
    pos, nt, past = [], [], n_past
    for start in range(0, n_tokens, bs):
        n = min(bs, n_tokens - start)
        p = max(0, min(n_ctx - n, past))
        pos += [p + i for i in range(n)]
        nt += [p + n] * n
        past += n
    return pos, nt


def pack(lib, slots, lengths, n_past, batch_size, n_ctx):
    n = len(slots)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    total = int(off[-1])
    out = np.zeros((max(total, 1), 5), np.int32)
    arr = lambda v: (C.c_int * max(len(v), 1))(*[int(x) for x in v])
    got = lib.ctb_multi_pack(n, arr(slots), arr(off), arr(n_past), batch_size, n_ctx, out.ctypes.data_as(C.POINTER(C.c_int)), len(out))
    assert got == total
    return out[:total]


def check(lib, slots, lengths, n_past, batch_size, n_ctx, exact_count=True):
    out = pack(lib, slots, lengths, n_past, batch_size, n_ctx)
    for s, m, p in zip(slots, lengths, n_past):
        rows = out[out[:, 0] == s]
        pos, nt = batch_eval_list(m, p, batch_size, n_ctx)
        assert rows[:, 1].tolist() == pos and rows[:, 2].tolist() == nt, (s, batch_size)
        assert rows[:, 4].tolist() == [0] * (m - 1) + [1] * (m > 0)
        assert (np.diff(rows[:, 3]) >= 0).all()                            # never in an earlier launch than the token before
        for a, b in zip(rows[:-1], rows[1:]):                                # one launch holds a slot's consecutive positions only
            assert a[3] != b[3] or b[1] == a[1] + 1
    launch = out[:, 3]
    assert (np.diff(launch) >= 0).all() and (launch.size == 0 or launch[0] == 0)
    assert np.bincount(launch).max(initial=0) <= PB_T
    if exact_count and len(out):
        assert launch[-1] + 1 == -(-len(out) // PB_T)
    return out


@pytest.mark.parametrize("batch_size", [1, 3, 5, 8, 64, 512])
def test_pack_matches_batch_eval(lib, batch_size):
    rng = np.random.default_rng(batch_size)
    lengths = [1, 2, 7, 31, 32, 33, 70] + rng.integers(1, 90, 25).tolist()
    slots = rng.permutation(32).tolist()
    n_past = rng.integers(0, 300, 32).tolist()
    check(lib, slots, lengths, n_past, batch_size, 512)


def test_pack_lockstep_decode_is_one_launch(lib):
    for s in (1, 2, 17, 32):
        out = check(lib, list(range(s)), [1] * s, list(range(100, 100 + s)), 8, 512)
        assert (out[:, 3] == 0).all() and (out[:, 2] == out[:, 1] + 1).all()


def test_pack_mixes_prompts_with_decode_tokens(lib):
    out = check(lib, [3, 0, 5], [1, 40, 1], [17, 0, 250], 64, 512)
    assert out[:, 3].tolist() == [0] * 32 + [1] * 10
    assert out[0].tolist() == [3, 17, 18, 0, 1] and out[-1].tolist() == [5, 250, 251, 1, 1]


@pytest.mark.parametrize("batch_size", [3, 8, 64])
def test_pack_n_past_clamp(lib, batch_size):
    """Past the context, every chunk is clamped to end at n_ctx, so a slot evaluates positions again: such a token starts a new
    launch (its K / V overwrite rows the earlier tokens read)."""
    n_ctx = 96
    out = check(lib, [0, 1], [40, 20], [80, 90], batch_size, n_ctx, exact_count=False)
    assert out[:, 1].max() == n_ctx - 1
    rows = out[out[:, 0] == 0]
    assert rows[:, 1].tolist() == batch_eval_list(40, 80, batch_size, n_ctx)[0]


def test_pack_empty_and_bad_offsets(lib):
    assert len(pack(lib, [0, 1], [0, 0], [0, 5], 8, 64)) == 0
    out = (C.c_int * 5)()
    assert lib.ctb_multi_pack(2, (C.c_int * 2)(0, 1), (C.c_int * 3)(0, 3, 1), (C.c_int * 2)(0, 0), 8, 64, out, 1) == 0


def test_create_without_gpu_is_refused(lib, tmp_models):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ctransformers_b200 import MultiLLM, synth
    from ctransformers_b200.lib import ConfigStruct
    path = tmp_models / "multi_nogpu.gguf"
    synth.write_llama(path, synth.LlamaShape(n_vocab=512, n_embd=256, n_head=4, n_head_kv=4, n_ff=512, n_layer=1), "Q4_K_M")
    assert lib.ctb_multi_create(str(path).encode(), b"gguf", ConfigStruct(64, 0, True, False), 4) is None
    with pytest.raises(RuntimeError):
        MultiLLM(str(path), n_slots=4)
