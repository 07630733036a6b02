"""Host-side check (no GPU) of how the paired decode-step kernel splits an input's staging between the two CTAs of a cluster
(csrc/matvec.cuh pair_block0, csrc/stream.cuh step_pair_fits), through ctb_stage_pair_split.  The device code uses the same
functions."""
import ctypes as C

import pytest

ST_NT = 320   # consumer threads of a step-kernel CTA (stream.cuh ST_NT)


def split(lib, K):
    b = (C.c_int * 3)()
    fits = lib.ctb_stage_pair_split(K, b)
    return fits, list(b)


@pytest.mark.parametrize("K", [256, 512, 768, 2816, 4096, 4608, 5120, 11008, 13824, 18176, 18432, 20480])
def test_every_block_once_rank0_takes_the_odd_one(lib, K):
    fits, (b0, b1, end) = split(lib, K)
    nb = K // 256
    assert (b0, end) == (0, nb)
    owner = [0] * b1 + [1] * (end - b1)
    assert len(owner) == nb and owner == sorted(owner)   # whole blocks, contiguous, rank 0 first
    assert b1 - b0 == (nb + 1) // 2 and end - b1 == nb // 2
    assert fits == 1, "every width up to 80 blocks fits two groups of 16 elements per thread"
    assert (b1 - b0) * 16 <= 2 * ST_NT


def test_widths_past_two_groups_per_thread_stay_unpaired(lib):
    assert split(lib, 20480)[0] == 1       # 80 blocks: rank 0 holds 40 = 640 groups of 16 = two per thread
    assert split(lib, 20736)[0] == 0       # 81 blocks: rank 0 would need a third
    assert split(lib, 300)[0] == -1        # not a whole number of blocks
