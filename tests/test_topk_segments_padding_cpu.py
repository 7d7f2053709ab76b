"""CPU check of the segment top-k oracle's padding (tests/test_gpu_topk_segments.py): for every dtype and direction the padding
key is the decode of the all-ones radix image, the value the C header names, and it sorts last against oraclelib's order,
NaNs and +-0 included."""
import numpy as np
import pytest

from tests import oraclelib
from tests.test_gpu_topk import TYPES, width
from tests.test_gpu_topk_segments import pad_key

# (dtype, largest) -> the padding's bit pattern, as osb200_topk_segments documents it
TABLE = {
    ("u16", False): 0xFFFF, ("u16", True): 0,
    ("i16", False): 0x7FFF, ("i16", True): 0x8000,
    ("f16", False): 0x7FFF, ("f16", True): 0xFFFF,
    ("bf16", False): 0x7FFF, ("bf16", True): 0xFFFF,
    ("u32", False): 0xFFFFFFFF, ("u32", True): 0,
    ("i32", False): 0x7FFFFFFF, ("i32", True): 0x80000000,
    ("f32", False): 0x7FFFFFFF, ("f32", True): 0xFFFFFFFF,
    ("u64", False): (1 << 64) - 1, ("u64", True): 0,
    ("i64", False): (1 << 63) - 1, ("i64", True): 1 << 63,
    ("f64", False): (1 << 63) - 1, ("f64", True): (1 << 64) - 1,
}


def _specials(t):
    """bit patterns of zeros, NaNs, infinities, extremes and a few random keys of dtype t"""
    c = TYPES[t][1]
    w = width(t)
    top = (1 << w) - 1
    vals = [0, 1, top, top - 1, 1 << (w - 1), (1 << (w - 1)) - 1, (1 << (w - 1)) + 1]
    if TYPES[t][3] == "f":
        ebits = {16: 5 if t == "f16" else 8, 32: 8, 64: 11}[w]
        inf = ((1 << ebits) - 1) << (w - 1 - ebits)
        vals += [inf, inf | (1 << (w - 1)), inf | 1, inf | 1 | (1 << (w - 1))]  # +-inf, +-NaN with a small payload
    rng = np.random.default_rng(w)
    return np.concatenate([np.array(vals, dtype=np.uint64).astype(c), rng.integers(0, np.iinfo(c).max, 64, dtype=c, endpoint=True)])


@pytest.mark.parametrize("largest", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
def test_padding_is_the_decoded_all_ones_image_and_sorts_last(t, largest):
    c = TYPES[t][1]
    kind = TYPES[t][3]
    pad = pad_key(t, largest)
    assert int(pad) == TABLE[(t, largest)]
    # oraclelib works on 32- and 64-bit containers: widen 16-bit keys into the top half of a uint32 (order-preserving)
    wide = np.uint32 if width(t) <= 32 else np.uint64
    shift = wide(32 - width(t)) if width(t) < 32 else wide(0)

    def image(bits):
        return oraclelib.to_radix((bits.astype(wide) << shift).astype(wide), kind, largest)

    ones = np.array([np.iinfo(wide).max], dtype=wide)
    dec = oraclelib.from_radix(ones, kind, largest)
    if width(t) < 32:
        assert int(dec[0] >> shift) == int(pad)
    else:
        assert int(dec[0]) == int(pad)
    keys = _specials(t)
    img = image(keys)
    pimg = image(np.array([pad], dtype=c))[0]
    assert (img <= pimg).all(), "a key sorts after the padding"
    others = keys[keys != pad]
    assert (image(others) < pimg).all()
