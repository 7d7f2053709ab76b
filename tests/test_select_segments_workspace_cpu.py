"""CPU checks of the segment select's long-path workspace (osb200_select_segments): the bound the header states, restated
here, is the library's host function osb200_select_segments_workspace_words (the layout the call checks) and the Python
package's select_segments_workspace; it depends on the shapes only, and it fits the alternate payloads (max_n 32-bit words)
of every handle with max_n >= max(n, num_segments) outside the test hook.  The call clamps max_segment_len to n, so with
n <= C (16,384, or 8,192 for 8-byte keys) the long path never runs and the bound is 0."""
import pytest

TILE = 8192


def round4(w):
    return (w + 3) // 4 * 4


def header_bound(n, num_segments, num_ranks, key_bytes, indices, long_min=None):
    """W of include/onesweep_b200.h, in 32-bit words"""
    long_min = long_min or (8192 if key_bytes == 8 else 16384) + 1
    if n < long_min or num_segments == 0:
        return 0
    listed = min(n // long_min, num_segments)
    tiles = -(-n // TILE) + listed
    w = round4(16 + listed * num_ranks * 260) + round4(listed) + 2 * round4(listed + 1)
    if indices:
        w += round4(tiles * num_ranks) + round4(-(-tiles // 16) + listed)
    return w


SHAPES = [(n, s) for n in (0, 1, 8192, 8193, 16384, 16385, 16386, 32770, 151_936, 1 << 20, (1 << 26) + 5, 1 << 32)
          for s in (1, 2, 3, 100, 151_936, 1 << 20)]


@pytest.mark.parametrize("key_bytes", [2, 4, 8])
def test_python_helper_and_host_function_are_the_header_bound(key_bytes):
    import gpusorting_b200 as g

    host = g.lib.osb200_select_segments_workspace_words
    for n, s in SHAPES:
        for r in (1, 3, 16):
            for ind in (False, True):
                want = header_bound(n, s, r, key_bytes, ind)
                assert host(n, s, r, key_bytes, int(ind)) == want, (n, s, r, ind)
                assert g.select_segments_workspace(n, s, r, key_bytes, ind) == want, (n, s, r, ind)
    assert host(1 << 20, 10, 0, 4, 1) == 0 and host(1 << 20, 10, 17, 4, 1) == 0 and host(1 << 20, 10, 1, 3, 1) == 0


@pytest.mark.parametrize("key_bytes", [2, 4, 8])
def test_bound_fits_every_handle_of_the_required_shape(key_bytes):
    cap = 8192 if key_bytes == 8 else 16384
    for n, s in SHAPES:
        for r in (1, 16):
            for ind in (False, True):
                assert header_bound(n, s, r, key_bytes, ind) <= max(n, s), (n, s, r, ind)
    # the tightest case: one long segment of C + 1 keys, 16 ranks, positions
    assert header_bound(cap + 1, 1, 16, key_bytes, True) <= cap + 1
    # about 0.52 words per key at most: 16 ranks over segments of C + 1 keys each
    n = 1000 * (cap + 1)
    assert header_bound(n, 1000, 16, key_bytes, True) <= 0.52 * n


def test_bound_grows_with_the_long_segments_only():
    # below C + 1 keys nothing can take the long path, whatever max_segment_len says
    assert header_bound(16384, 2, 16, 4, True) == 0 and header_bound(10, 2, 16, 4, True) == 0 and header_bound(0, 2, 1, 8, True) == 0
    assert header_bound(8193, 1, 16, 8, True) > 0
    # the test hook (long_min = 2) is bounded by the number of segments
    assert header_bound(1 << 20, 100, 16, 4, False, long_min=2) == round4(16 + 100 * 16 * 260) + 100 + 2 * 104
