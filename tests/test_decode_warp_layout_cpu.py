"""The state_len 3 decode runs each chunk in one warp, lane l holding states l and l + 32 (decode.cu, crf_decode_warp_kernel).
Its posterior normaliser must add in the order of the contract (oracle/crf_oracle.c posts_row): groups of 32 consecutive
states, an xor butterfly within each group, groups added left to right.  These tests emulate the warp's order in float32
and hold it to posts_row's order bit for bit, and show that the order is not free: pairing states 2l and 2l + 1 on a lane
gives different sums."""
import numpy as np

S = 64


def _posts_row_z(e):
    """posts_row's normaliser for S = 64 (one state per part, G = 32)."""
    part = e.astype(np.float32).copy()
    o = 16
    while o >= 1:
        part = (part + part[np.arange(S) ^ o]).astype(np.float32)
        o >>= 1
    return np.float32(part[0] + part[32])


def _warp_z(lo, hi):
    """Lane l holds lo[l] and hi[l]: one xor butterfly over the lanes for each, then z0 + z1 (every lane ends equal)."""
    z0, z1 = lo.astype(np.float32).copy(), hi.astype(np.float32).copy()
    lanes = np.arange(32)
    o = 16
    while o >= 1:
        z0 = (z0 + z0[lanes ^ o]).astype(np.float32)
        z1 = (z1 + z1[lanes ^ o]).astype(np.float32)
        o >>= 1
    assert (z0 == z0[0]).all() and (z1 == z1[0]).all()
    return (z0 + z1).astype(np.float32)


def _rows(seed, n=2000):
    rng = np.random.default_rng(seed)
    rows = [np.exp(rng.standard_normal(S).astype(np.float32) * 3.0 - 4.0).astype(np.float32) for _ in range(n)]
    for _ in range(200):   # ties: a few distinct values repeated, and a row of ones (the maximum state has e = 1)
        vals = np.exp(-rng.random(3).astype(np.float32) * 5.0).astype(np.float32)
        rows.append(vals[rng.integers(3, size=S)])
    rows.append(np.ones(S, np.float32))
    return rows


def test_lanes_l_and_l_plus_32_match_posts_row_order():
    for e in _rows(1):
        z = _warp_z(e[:32], e[32:])
        ref = _posts_row_z(e)
        assert (z.view(np.uint32) == ref.view(np.uint32)).all()


def test_pairing_adjacent_states_changes_the_sum():
    differs = 0
    for e in _rows(2):
        z = _warp_z(e[0::2], e[1::2])[0]
        differs += z.view(np.uint32) != _posts_row_z(e).view(np.uint32)
    assert differs > 0
