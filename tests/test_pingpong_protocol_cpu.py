"""Model of the ping-pong turn protocol of the narrow tensor-core MLP kernels (bwd_blk_body in mlp_bwd_tc.cu,
fwd_rs_body in mlp_fwd_tc.cu): the two warpgroups of a CTA hand a token back and forth through named barriers
3 and 4 (256 threads: one warpgroup's bar.sync and the other's bar.arrive).

The barrier sequence of each warpgroup is generated from the same tile counts and conditions as the kernels,
then every interleaving of the two warpgroups is explored with the hardware's counting semantics (a barrier
generation completes when 256 threads, two warpgroup arrivals, have reached it).  Checked: no reachable state
is stuck (no circular wait; both warpgroups reach the closing __syncthreads), every generation is completed
by one warpgroup of each side (an arrival of the same warpgroup twice would release the barrier without the
other), and every barrier is back at zero at the end - so the closing __syncthreads and the grid barrier are
never reached with a token in flight.
"""
import pytest

TURN0, TURN1 = 3, 4  # turn barrier of warpgroup 0 / 1


def bwd_ops(num_tiles, cpg, r):
    """Per-warpgroup barrier ops of bwd_blk_body for CTA r of a group of cpg (tiles r, r + cpg, ... alternate):
    one turn per tile, around the GEMM2 issue."""
    seqs = []
    for wg in (0, 1):
        own, other = TURN0 + wg, TURN1 - wg
        ops = []
        tile = r + cpg * wg
        while tile < num_tiles:
            if wg == 1 or tile != r:
                ops.append(("sync", own))
            if wg == 0 or tile + cpg < num_tiles:
                ops.append(("arrive", other))
            tile += 2 * cpg
        ntiles = (num_tiles - 1 - r) // cpg + 1 if r < num_tiles else 0
        if wg == 1 and ntiles % 2 == 1:
            ops.append(("sync", own))
        ops.append(("sync", 0))  # closing __syncthreads
        seqs.append(ops)
    return seqs


def fwd_ops(num_tiles, ncta, cta, nslices, npass=1):
    """Per-warpgroup barrier ops of fwd_rs_body for CTA cta of ncta (warpgroup unit 2 cta + wg, stride 2 ncta)."""
    nunits, nb = 2 * ncta, (nslices + 1) // 2
    seqs = []
    for wg in (0, 1):
        unit = 2 * cta + wg
        ops = []
        for _ in range(npass):
            ops += [("sync", 0), ("sync", 0)]  # the pass's weight staging
            tile = unit
            while tile < num_tiles:
                for b in range(nb):
                    first, last = b == 0, b == nb - 1
                    if wg == 1 or not (tile == unit and first):
                        ops.append(("sync", TURN0 + wg))
                    if wg == 0 or not last or tile - 1 + nunits < num_tiles:
                        ops.append(("arrive", TURN1 - wg))
                tile += nunits
            if wg == 1 and tile - 1 < num_tiles:
                for b in range(nb):
                    ops.append(("sync", TURN1))
                    if b + 1 < nb:
                        ops.append(("arrive", TURN0))
        seqs.append(ops)
    return seqs


def explore(seqs):
    """Every interleaving of the two warpgroups' ops; raises AssertionError on a hazard or a stuck state."""
    # state: (pc0, pc1, waiting0, waiting1, barriers) with barriers a tuple of (id, arrivals) for the
    # barriers with a partial generation; waiting = the barrier a warpgroup is blocked on, or -1
    start = (0, 0, -1, -1, ())
    seen, stack = {start}, [start]
    while stack:
        pc0, pc1, w0, w1, bars = stack.pop()
        pcs, waits = [pc0, pc1], [w0, w1]
        if pcs[0] == len(seqs[0]) and pcs[1] == len(seqs[1]):
            assert bars == (), f"barriers left with arrivals at the end: {bars}"
            continue
        moved = False
        for wg in (0, 1):
            if waits[wg] != -1 or pcs[wg] == len(seqs[wg]):
                continue
            kind, bid = seqs[wg][pcs[wg]]
            partial = dict(bars)
            arrivals = partial.get(bid, ()) + (wg,)
            npcs, nwaits = list(pcs), list(waits)
            npcs[wg] += 1
            if len(arrivals) == 2:
                assert arrivals[0] != arrivals[1], f"barrier {bid} completed by warpgroup {wg} alone"
                partial.pop(bid, None)
                nwaits = [-1 if x == bid else x for x in nwaits]  # the generation releases its waiters
            else:
                partial[bid] = arrivals
                if kind == "sync":
                    nwaits[wg] = bid
            state = (npcs[0], npcs[1], nwaits[0], nwaits[1], tuple(sorted(partial.items())))
            moved = True
            if state not in seen:
                seen.add(state)
                stack.append(state)
        assert moved, f"stuck: warpgroups at ops {pcs} of {[len(s) for s in seqs]}, waiting on {waits}, {bars}"
    return len(seen)


def test_model_catches_an_unbalanced_protocol():
    # warpgroup 1 releasing the token after its last turn as well: nobody awaits that arrival
    seqs = bwd_ops(2, 1, 0)
    bad = [seqs[0], seqs[1][:-1] + [("arrive", TURN0), ("sync", 0)]]
    with pytest.raises(AssertionError):
        explore(bad)
    # two arrivals of warpgroup 0 in a row complete barrier 4 without warpgroup 1
    with pytest.raises(AssertionError):
        explore([[("arrive", TURN1), ("arrive", TURN1), ("sync", 0)], [("sync", TURN1), ("sync", 0)]])
    # warpgroup 1 without its padding turns: warpgroup 0 waits for ever
    seqs = bwd_ops(1, 1, 0)
    with pytest.raises(AssertionError):
        explore([seqs[0], [("sync", 0)]])


@pytest.mark.parametrize("cpg", range(1, 6))
def test_bwd_small_counts(cpg):
    # 0, 1, 2 and more tiles per warpgroup, every CTA of the group
    for num_tiles in range(0, 4 * cpg + 2):
        for r in range(cpg):
            explore(bwd_ops(num_tiles, cpg, r))


# batch rows per network: c3, c4 and c5 (T x B and (T + 1) x B), the pair shapes of test_gpu_bwd_blocks.py
# (35 / 42, 150 / 200, 903 / 1032, 8196 / 10245), its single shapes (5, 64, 65, 6401, 86017) and the tile
# edges and odd batches of test_gpu_mlp_corners.py (1, 31, 32, 33, 63, 777, 1000, 4097)
SHAPE_ROWS = [20480, 21504, 81920, 86016, 819200, 35, 42, 150, 200, 903, 1032, 8196, 10245, 5, 64, 65, 6401, 86017,
              1, 31, 32, 33, 63, 777, 1000, 4097]


@pytest.mark.parametrize("rows", SHAPE_ROWS)
def test_bwd_shapes(rows):
    num_tiles = (rows + 63) // 64
    # CTAs per hidden block: whatever split_sets gives on 132 SMs (at most 66 for H = 128)
    for cpg in range(1, 67):
        if num_tiles > 2000 and cpg % 4 != 1:
            continue
        for r in range(cpg):
            explore(bwd_ops(num_tiles, cpg, r))


@pytest.mark.parametrize("nslices", [1, 2, 3, 4, 7, 8])
def test_fwd_small_counts(nslices):
    for ncta in range(1, 4):
        for num_tiles in range(0, 4 * ncta + 3):
            for cta in range(ncta):
                explore(fwd_ops(num_tiles, ncta, cta, nslices))
                explore(fwd_ops(num_tiles, ncta, cta, nslices, npass=2))


@pytest.mark.parametrize("rows", SHAPE_ROWS)
def test_fwd_shapes(rows):
    num_tiles = (rows + 63) // 64
    for ncta in (1, 2, 3, 66, 131):
        for cta in sorted({0, 1, ncta // 2, ncta - 1}):
            if cta < ncta:
                explore(fwd_ops(num_tiles, ncta, cta, 8))  # H = 256: 4 batches per tile
