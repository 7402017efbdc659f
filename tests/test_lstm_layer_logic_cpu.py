"""CPU model of the gate-row permutation and fragment ownership of lstm_layer_kernel (dorado_b200/csrc/lstm_model.cu, the
fused LSTM layer of lstm_size 96).  The kernel's results are checked against the numpy oracle on the GPU
(tests/test_forward_gpu.py); this test pins the reasoning that lets its gate math run from registers: after the host permutes
the gate rows, the m16n8k16 accumulators of every thread hold all four gates of its cells, and every (gate, unit, chunk) has
exactly one owner."""
C = 96      # FL_C
NB = 16     # FL_NB: chunks per CTA
WARPS = C // 8


def lstm_fused_row(gate, unit):
    """lstm_model.cu lstm_fused_row: permuted row of PyTorch gate row gate * C + unit."""
    return (unit // 8) * 32 + gate * 8 + unit % 8


def accumulator_owner(row, col):
    """(warp, lane, tile, n tile, element) that holds D[row][col] of the warp-stacked m16n8k16 tiles (tc.cuh: c[4] = rows
    lane / 4 (+ 8) x columns 2 (lane % 4) + {0, 1}), warp w covering rows 32 w .. 32 w + 31 as two m16 tiles."""
    warp, r = divmod(row, 32)
    tile, r = divmod(r, 16)
    half, r = divmod(r, 8)
    nt, c = divmod(col, 8)
    return warp, r * 4 + c // 2, tile, nt, 2 * half + c % 2


def test_permutation_is_a_bijection():
    rows = [lstm_fused_row(g, u) for g in range(4) for u in range(C)]
    assert sorted(rows) == list(range(4 * C))


def test_every_gate_has_one_owner_and_owners_hold_whole_cells():
    owners = {}
    for g in range(4):
        for u in range(C):
            for n in range(NB):
                o = accumulator_owner(lstm_fused_row(g, u), n)
                assert o not in owners, (g, u, n)
                owners[o] = (g, u, n)
    assert len(owners) == 4 * C * NB

    # the kernel reads gate g of its cell (n tile nt, chunk of the pair e) from tile g // 2, element 2 (g % 2) + e, for unit
    # 8 warp + lane / 4 and chunk 8 nt + 2 (lane % 4) + e
    cells = set()
    for warp in range(WARPS):
        for lane in range(32):
            unit = warp * 8 + lane // 4
            for nt in range(2):
                for e in range(2):
                    chunk = nt * 8 + 2 * (lane % 4) + e
                    for g in range(4):
                        assert owners[(warp, lane, g // 2, nt, 2 * (g % 2) + e)] == (g, unit, chunk)
                    cells.add((unit, chunk))
    assert len(cells) == C * NB
