"""CPU models of pieces of integer logic inside dorado_b200/csrc/decode.cu and gemm.cu, checked against the straightforward form the
reference uses.  The kernels themselves are pinned bit for bit against the C oracle on the GPU (tests/test_decode_gpu.py,
tests/test_full_size_gpu.py); these tests pin the *reasoning* behind the two rewrites, including the rare paths real data
seldom reaches (equal hashes inside a beam, hash-table slots shared by several lanes, a table full of stale entries).

1. beam_step's stay / step merge (beam_search.cpp:264-305): the reference compares every stay against every step of the same
   base.  The kernel computes, per stay, the one hash its merging step's parent must have (inverse CRC), looks that hash up in a
   1024-entry lane-id table over the low hash bits, and broadcasts the lanes whose own table entry was overwritten.
2. kmer_block_prob's duplicate elimination (beam_search.cpp:459-503): the reference adds the posteriors of the state's eight
   shift neighbours, skipping a neighbour equal to the state or to an earlier neighbour (36 compares); the kernel only makes
   the 24 compares that can be true.
"""
import random

SLOTS = 1024
POLY = 0x82F63B78


def crc2(crc, nb):
    b = (nb ^ crc) & 1
    crc = (crc >> 1) ^ (POLY if b else 0)
    b = ((nb >> 1) ^ crc) & 1
    crc = (crc >> 1) ^ (POLY if b else 0)
    return crc & 0xFFFFFFFF


def crc2_inv(crc, nb):
    b = crc >> 31
    t = crc ^ (POLY if b else 0)
    crc = ((t << 1) & 0xFFFFFFFF) | (b ^ ((nb >> 1) & 1))
    b = crc >> 31
    t = crc ^ (POLY if b else 0)
    crc = ((t << 1) & 0xFFFFFFFF) | (b ^ (nb & 1))
    return crc


def kernel_lookup(hashes, states, width, table, rng):
    """decode.cu beam_step, merge lookup: returns (any equal hashes, matching parent lane per stay or -1)"""
    valid = [l < width for l in range(32)]
    vmask = (1 << width) - 1
    target = [crc2_inv(hashes[l], states[l] & 3) for l in range(32)]
    own = [hashes[l] & (SLOTS - 1) for l in range(32)]
    order = list(range(32))
    rng.shuffle(order)  # which lane's byte store survives in a shared slot is not defined
    for l in order:
        if valid[l]:
            table[own[l]] = l
    rb = [table[own[l]] if valid[l] else l for l in range(32)]
    c = [table[target[l] & (SLOTS - 1)] & 31 for l in range(32)]
    overwritten = [valid[l] and rb[l] != l for l in range(32)]
    jm = [-1] * 32
    dup = False
    for l in range(32):
        if valid[l] and ((vmask >> c[l]) & 1) and hashes[c[l]] == target[l]:
            jm[l] = c[l]
    for j in range(32):
        if overwritten[j]:
            for l in range(32):
                if valid[l] and l != j and hashes[l] == hashes[j]:
                    dup = True
                if valid[l] and target[l] == hashes[j]:
                    jm[l] = j
    return dup, jm


def test_crc2_inverse():
    rng = random.Random(3)
    for _ in range(20000):
        h, nb = rng.getrandbits(32), rng.getrandbits(2)
        assert crc2_inv(crc2(h, nb), nb) == h


def test_table_merge_lookup_equals_all_pairs_search():
    rng = random.Random(1)
    table = [rng.randrange(256) for _ in range(SLOTS)]  # never cleared in the kernel: start from garbage
    dups = matches = shared = 0
    for _ in range(60000):
        width = rng.choice([1, 2, 5, 17, 31, 32])
        mode = rng.random()
        hashes = [rng.getrandbits(32) for _ in range(32)]   # lanes >= width hold stale values
        states = [rng.getrandbits(6) for _ in range(32)]
        if mode < 0.5:     # parent / child pairs: lane b is lane a's sequence plus b's newest base
            for _ in range(rng.randrange(1, 8)):
                a, b = rng.randrange(width), rng.randrange(width)
                if a != b:
                    hashes[b] = crc2(hashes[a], states[b] & 3)
        if mode < 0.25:    # different hashes in the same table slot
            for _ in range(rng.randrange(1, 6)):
                a, b = rng.randrange(width), rng.randrange(width)
                if a != b:
                    hashes[b] = (hashes[b] & ~(SLOTS - 1)) | (hashes[a] & (SLOTS - 1))
                    shared += 1
        if 0.4 < mode < 0.5:  # equal hashes: the case that must be handed to the sequential replay
            a, b = rng.randrange(width), rng.randrange(width)
            if a != b:
                hashes[b] = hashes[a]
        dup, jm = kernel_lookup(hashes, states, width, table, rng)
        assert dup == (len(set(hashes[:width])) != width)
        if dup:
            dups += 1
            continue
        for i in range(width):
            t = crc2_inv(hashes[i], states[i] & 3)
            hits = [j for j in range(width) if hashes[j] == t]
            assert jm[i] == (hits[0] if hits else -1)
            matches += bool(hits)
    assert dups > 1000 and matches > 10000 and shared > 10000


def test_kmer_neighbour_deduplication():
    for state_len in (3, 4, 5):
        S = 1 << (2 * state_len)
        msb = S >> 2
        for state in range(S):
            l, r = state >> 2, (state << 2) & (S - 1)
            sh = []
            for b in range(4):
                sh += [l + msb * b, r + b]
            ref = [k for k in range(8) if sh[k] != state and all(sh[j] != sh[k] for j in range(k))]
            d = l - r
            got = []
            for b in range(4):
                L, R = l + msb * b, r + b
                if L != state and all(bb - msb * b != d for bb in range(b)):
                    got.append(2 * b)
                if R != state and all(b - msb * bb != d for bb in range(b + 1)):
                    got.append(2 * b + 1)
            assert got == ref, (state_len, state)


def test_gemm_tile_schedules_cover_every_tile_once():
    """gemm.cu gemm_tile_at + the grid rule of run_gemm: the persistent schedule (shorter dimension fastest, CTAs take
    consecutive tiles, grid = min(tiles, max_ctas)) visits every (row tile, column tile) exactly once."""
    def tiles_of(cta, grid, m_tiles, n_tiles, mfast):
        i = 0
        while True:
            tile = cta + i * grid
            if tile >= m_tiles * n_tiles:
                return
            yield (tile % m_tiles, tile // m_tiles) if mfast else (tile // n_tiles, tile % n_tiles)
            i += 1

    for m_tiles, n_tiles in [(12, 3332), (832, 12), (832, 32), (7, 6), (1, 5), (300, 1)]:
        for max_ctas in (132, 100, 37):
            grid = min(m_tiles * n_tiles, max_ctas)
            seen = {}
            for cta in range(grid):
                for t in tiles_of(cta, grid, m_tiles, n_tiles, m_tiles < n_tiles):
                    seen[t] = seen.get(t, 0) + 1
            assert len(seen) == m_tiles * n_tiles and set(seen.values()) == {1}, (m_tiles, n_tiles, max_ctas)
