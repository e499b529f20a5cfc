"""The small-source path of take_bytes (Dictionary<Int32,Utf8> -> Utf8 = take(dictionary values, keys),
arrow-cast/src/cast/dictionary.rs:310-317; take_bytes arrow-select/src/take.rs:499-627): dictionary table in shared memory
(k_dict_table / k_dict_block_totals / k_dict_copy) vs the oracle, around its eligibility limits — D up to 8192 entries of at
most 16 bytes, >= 65536 keys — and the fallbacks (an entry of 17 bytes, D = 8193)."""
import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import HostArray

pytestmark = pytest.mark.gpu


def make_dict(rng, d, max_len, null_p=None):
    lens = rng.integers(0, max_len + 1, d)
    offs = np.zeros(d + 1, dtype=np.int32)
    offs[1:] = np.cumsum(lens)
    data = rng.integers(1, 256, int(offs[-1]) + 16).astype(np.uint8)
    if null_p is None:
        nulls = HostArray(acu.U8, np.zeros(0, np.uint8), d, None, 0, 0, 0)
    else:
        mask = rng.random(d) >= null_p
        nulls = HostArray(acu.U8, np.zeros(0, np.uint8), d, acu.pack_bits(mask), 0, 0, int(d - mask.sum()))
    return offs, data, nulls


def check(gpu, oracle, offs, data, nulls, keys, what):
    g, e = gpu.take_bytes(offs, data, nulls, keys), oracle.take_bytes(offs, data, nulls, keys)
    assert np.array_equal(g[0], e[0]), f"{what}: offsets"
    assert np.array_equal(g[1], e[1]), f"{what}: value bytes"
    assert (g[2].validity is None) == (e[2].validity is None) and g[2].null_count == e[2].null_count, f"{what}: nulls"
    if e[2].validity is not None:
        assert np.array_equal(g[2].valid_mask(), e[2].valid_mask())


@pytest.mark.parametrize("d,max_len", [(1, 16), (100, 12), (4096, 12), (8192, 16), (8193, 8), (500, 17), (300, 0)])
def test_dictionary_gather(gpu, oracle, d, max_len):
    rng = np.random.default_rng(d * 31 + max_len)
    for m in (65536, 65537, 131072 + 2048, 200_001):
        for key_null_p, dict_null_p in [(None, None), (0.05, None), (0.1, 0.2)]:
            offs, data, nulls = make_dict(rng, d, max_len, dict_null_p)
            keys_v = rng.integers(0, d, m).astype(np.int32)
            mask = None if key_null_p is None else rng.random(m) >= key_null_p
            keys = HostArray.from_numpy(abi.I32, keys_v, mask)
            check(gpu, oracle, offs, data, nulls, keys, f"D={d} L<={max_len} m={m} nulls={key_null_p}/{dict_null_p}")


def test_dictionary_gather_out_of_bounds_key(gpu, oracle):
    rng = np.random.default_rng(3)
    offs, data, nulls = make_dict(rng, 64, 8)
    m = 100_000
    keys_v = rng.integers(0, 64, m).astype(np.int32)
    keys_v[77_777] = 64
    mask = np.ones(m, dtype=bool)
    keys = HostArray.from_numpy(abi.I32, keys_v, None)
    with pytest.raises(acu.ArrowError) as ge:
        gpu.take_bytes(offs, data, nulls, keys)
    with pytest.raises(acu.ArrowError) as oe:
        oracle.take_bytes(offs, data, nulls, keys)
    assert ge.value.status == oe.value.status == abi.ERR_PANIC_OUT_OF_BOUNDS and ge.value.index == oe.value.index == 77_777
    mask[77_777] = False  # under a null key an out-of-bounds value is fine (zero-length slot)
    keys = HostArray.from_numpy(abi.I32, keys_v, mask)
    check(gpu, oracle, offs, data, nulls, keys, "oob under a null key")


def test_dictionary_gather_offset_overflow(gpu, oracle):
    """take.rs:520-523,561-574: the running total passes i32::MAX => Err(OffsetOverflowError(capacity)), here through the
    dictionary path (2^27 + 1000 keys of 16-byte entries), with the capacity the reference reports (the oracle's)."""
    d, m = 4, (1 << 27) + 1000
    offs = (np.arange(d + 1) * 16).astype(np.int32)
    data = np.full(d * 16 + 16, ord("x"), dtype=np.uint8)
    nulls = HostArray(acu.U8, np.zeros(0, np.uint8), d, None, 0, 0, 0)
    keys = HostArray.from_numpy(abi.I32, (np.arange(m, dtype=np.int64) % d).astype(np.int32), None)
    errs = []
    for be in (gpu, oracle):
        with pytest.raises(acu.ArrowError) as e:
            be.take_bytes(offs, data, nulls, keys)
        errs.append(e.value)
    assert errs[0].status == errs[1].status == abi.ERR_OFFSET_OVERFLOW
    assert str(errs[0]) == str(errs[1])


@pytest.mark.parametrize("d,per_sm", [(4096, 2), (8192, 1)])
def test_dictionary_gather_multi_round(gpu, oracle, d, per_sm):
    """k_dict_copy keeps per_sm CTAs resident per SM (its shared-memory table grows with D) and each CTA loops over 2048-row
    rounds, prefetching the next round's keys: sizes that give every CTA at least two rounds, with key and dictionary nulls."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m = 2 * sms * per_sm * 2048 + 1001
    rng = np.random.default_rng(d + 7)
    offs, data, nulls = make_dict(rng, d, 16, 0.2)
    keys_v = rng.integers(0, d, m).astype(np.int32)
    keys = HostArray.from_numpy(abi.I32, keys_v, rng.random(m) >= 0.05)
    check(gpu, oracle, offs, data, nulls, keys, f"D={d} m={m} over {sms} SMs")
