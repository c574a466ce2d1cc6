"""CPU model of the page bookkeeping of a rows-as-M MaxSim epilogue (patch rows as the MMA M operand, eight epilogue warps
that each see one chunk of a tile and meet in a page-slot table).

This file guards no shipped code: the CUDA kernel (maxsim_wgmma.cu) holds whole query groups per warp and has no slot table.
It pins the ALGORITHM of the rows-as-M design -- a pure-Python model, independent of CUDA -- for anyone who brings that
orientation back (it pays off where the MMA's smallest M is larger than one query's 32 tokens).  Its invariants:

  * every 8-tile block, a warp derives from two 32-bit masks (chunk exists / chunk starts a page) the ordinal of each page
    in the CTA's page sequence and the extent [start, end) of the page it is accumulating -- no page_start lookups;
  * a warp (lane quadrant q, set e) owns chunk q of the tiles with seq % 2 == e, keeps a running maximum per page and hands
    it to a table of kRmSlots page slots (slot = ordinal % kRmSlots) together with the number of chunks it saw; the warp
    whose contribution completes the page's chunk count emits the page and frees the slot;
  * a finished page is flushed at the next block at the latest, so with at most 8 tiles (the accumulator ring) between the
    fastest and the slowest warp no two live pages share a slot.

The model walks random ragged corpora with a random interleaving of the warps (bounded by the accumulator ring exactly like
the kernel: tile T can be drained only after every owner of tile T - 8 has drained it) and checks that every page is emitted
exactly once with the maximum over all of its chunks.
"""
import random

import pytest

K_SLOTS = 128   # kRmSlots
K_ACC = 8       # accumulator ring (tiles in flight between the MMA issuer and the slowest epilogue warp)


def build_stream(page_chunks, unit_chunks, rng):
    """The chunk stream of ONE CTA: whole pages grouped into units of ~unit_chunks chunks; every unit is padded to whole
    tiles (4 chunks) with invalid chunks (-1), exactly like the tail tile of a unit in the kernel."""
    units, cur = [], []
    for p, n in enumerate(page_chunks):
        if n == 0:
            continue  # zero-length pages own no chunks
        cur.extend([p] * n)
        if len(cur) >= unit_chunks:
            units.append(cur)
            cur = []
    if cur:
        units.append(cur)
    tiles = []  # (unit index, tile-in-unit t, [4 page ids or -1])
    for u, chunks in enumerate(units):
        padded = chunks + [-1] * (-len(chunks) % 4)
        for t in range(len(padded) // 4):
            tiles.append((u, t, padded[4 * t:4 * t + 4]))
    values = [[rng.randrange(-1000, 1000) if pg >= 0 else None for pg in tl[2]] for tl in tiles]
    return tiles, values


class Table:
    def __init__(self):
        self.pm = [None] * K_SLOTS   # running maximum per slot (None = INT_MIN)
        self.cnt = [0] * K_SLOTS
        self.owner = [None] * K_SLOTS  # model-only: which page currently uses the slot
        self.emitted = {}


class Warp:
    """One epilogue warp: lane quadrant `quad`, set `eset` (tiles with seq % 2 == eset)."""

    def __init__(self, quad, eset, tiles, values, table, totals):
        self.quad, self.eset, self.tiles, self.values, self.table, self.totals = quad, eset, tiles, values, table, totals
        self.seq = 0
        self.cp, self.cord, self.ccount, self.rm = -1, 0, 0, None
        self.g_base, self.last_change_g, self.cp_start_g, self.cp_end_g = 0, -1, 0, -1
        self.last_pg, self.ord_base, self.cmask, self.vmask = -1, 0, 0, 0
        self.block = []
        self.done = False

    # ---- the kernel's lambdas
    def flush(self):
        tb, slot = self.table, self.cord % K_SLOTS
        assert tb.owner[slot] in (None, self.cp), f"slot {slot} shared by pages {tb.owner[slot]} and {self.cp}"
        tb.owner[slot] = self.cp
        tb.pm[slot] = self.rm if tb.pm[slot] is None else max(tb.pm[slot], self.rm)
        old = tb.cnt[slot]
        tb.cnt[slot] += self.ccount
        total = self.cp_end_g - self.cp_start_g
        assert total == self.totals[self.cp], (self.cp, total, self.totals[self.cp])
        assert old + self.ccount <= total
        if old + self.ccount == total:
            assert self.cp not in tb.emitted, f"page {self.cp} emitted twice"
            tb.emitted[self.cp] = tb.pm[slot]
            tb.pm[slot], tb.cnt[slot], tb.owner[slot] = None, 0, None

    def adopt(self, pg, i):
        if self.cp >= 0:
            self.flush()
        upto = ((2 << i) - 1) & 0xFFFFFFFF
        le, gt = self.cmask & upto, self.cmask & ~upto & 0xFFFFFFFF
        self.cp, self.ccount, self.rm = pg, 0, None
        self.cord = self.ord_base + bin(le).count("1")
        self.cp_start_g = self.g_base + le.bit_length() - 1 if le else self.last_change_g
        self.cp_end_g = self.g_base + (gt & -gt).bit_length() - 1 if gt else -1

    def block_setup(self, first_tile):
        self.ord_base += bin(self.cmask).count("1")
        if self.cmask:
            self.last_change_g = self.g_base + self.cmask.bit_length() - 1
        self.g_base += bin(self.vmask).count("1")
        u = self.tiles[first_tile][0]
        cur = []
        for k in range(8):  # the 32 chunks of this block: tiles of the same unit only
            if first_tile + k < len(self.tiles) and self.tiles[first_tile + k][0] == u:
                cur.extend(self.tiles[first_tile + k][2])
            else:
                cur.extend([-1] * 4)
        self.block = cur
        prev = [self.last_pg] + cur[:-1]
        self.vmask = sum(1 << l for l in range(32) if cur[l] >= 0)
        self.cmask = sum(1 << l for l in range(32) if cur[l] >= 0 and cur[l] != prev[l])
        nv = bin(self.vmask).count("1")
        assert self.vmask == (1 << nv) - 1, "valid chunks must be a prefix of the block"
        self.last_pg = cur[nv - 1]
        if self.cp >= 0 and self.cp_end_g < 0 and self.cmask:
            self.cp_end_g = self.g_base + (self.cmask & -self.cmask).bit_length() - 1
        if self.cp >= 0 and 0 <= self.cp_end_g <= self.g_base:
            self.flush()
            self.cp = -1

    def step(self):
        """Process tile self.seq (block setup on the first tile of a block; drain only if this warp owns the tile)."""
        u, t, pages = self.tiles[self.seq]
        if t % 8 == 0:
            self.block_setup(self.seq)
        if self.seq % 2 == self.eset:
            i = 4 * (t % 8) + self.quad
            if (self.vmask >> i) & 1:
                pg = self.block[i]
                assert pg == pages[self.quad]
                if pg != self.cp:
                    self.adopt(pg, i)
                v = self.values[self.seq][self.quad]
                self.rm = v if self.rm is None else max(self.rm, v)
                self.ccount += 1
        self.seq += 1
        if self.seq == len(self.tiles):
            if self.cp >= 0:
                if self.cp_end_g < 0:
                    self.cp_end_g = self.g_base + bin(self.vmask).count("1")
                self.flush()
            self.done = True


def run_model(page_chunks, unit_chunks, seed, schedule="random"):
    rng = random.Random(seed)
    tiles, values = build_stream(page_chunks, unit_chunks, rng)
    if not tiles:
        return
    totals, want = {}, {}
    for tl, vs in zip(tiles, values):
        for pg, v in zip(tl[2], vs):
            if pg >= 0:
                totals[pg] = totals.get(pg, 0) + 1
                want[pg] = v if pg not in want else max(want[pg], v)
    table = Table()
    warps = [Warp(q, e, tiles, values, table, totals) for e in (0, 1) for q in range(4)]
    while not all(w.done for w in warps):
        # accumulator ring: tile T may be drained once every owner of tile T - K_ACC has drained it (= moved past it)
        def may_advance(w):
            if w.done:
                return False
            t_old = w.seq - K_ACC
            if t_old < 0:
                return True
            owners = [x for x in warps if x.eset == t_old % 2]
            return all(x.seq > t_old for x in owners)
        ready = [w for w in warps if may_advance(w)]
        assert ready, "model deadlock"
        if schedule == "run_ahead":    # the fastest warp runs as far ahead as the ring lets it
            w = max(ready, key=lambda x: (x.seq, rng.random()))
        elif schedule == "starve":     # one warp only moves when nobody else can
            others = [x for x in ready if x is not warps[seed % 8]]
            w = rng.choice(others) if others else ready[0]
        else:
            w = rng.choice(ready)
        w.step()
    assert table.emitted == want
    assert all(c == 0 for c in table.cnt) and all(o is None for o in table.owner)


@pytest.mark.parametrize("seed", range(6))
def test_uniform_1024_row_pages(seed):
    run_model([32] * 300, 128, seed)  # the BASELINE shape: a page = one 8-tile block, 4 pages per unit


@pytest.mark.parametrize("seed", range(12))
def test_ragged_pages_and_unit_sizes(seed):
    rng = random.Random(1000 + seed)
    pages = [rng.choice([0, 1, 1, 2, 3, 4, 5, 8, 9, 31, 32, 33, 40]) for _ in range(rng.randrange(1, 600))]
    run_model(pages, rng.choice([2, 4, 13, 32, 128]), seed)


@pytest.mark.parametrize("schedule", ["run_ahead", "starve"])
@pytest.mark.parametrize("seed", range(8))
def test_adversarial_interleavings_of_one_chunk_pages(seed, schedule):
    """Worst case for the slot table: every chunk is its own page (32 new pages per block) while one warp lags the full depth of
    the accumulator ring behind the others."""
    rng = random.Random(77 + seed)
    pages = [1] * 700 + [rng.choice([1, 2, 5]) for _ in range(300)]
    run_model(pages, rng.choice([4, 32, 128]), seed, schedule)


@pytest.mark.parametrize("seed", range(4))
def test_quadrants_without_rows_for_hundreds_of_pages(seed):
    """A 4-chunk page followed by hundreds of 1-2 chunk pages in 2-chunk units: lane quadrants 2 and 3 see no rows for > kRmSlots
    pages.  Without the flush of finished pages at the next block the slot table wraps around under them (the GPU test of the
    same shape is test_rows_as_m_kernel_flushes_finished_pages_early)."""
    rng = random.Random(seed)
    pages = [4] + [rng.choice([1, 2]) for _ in range(500)] + [4] + [2] * 300
    run_model(pages, 2, seed)


def test_model_detects_a_wrapping_slot_table():
    """The same corner case with the early flush disabled must trip the model's slot-sharing assertion -- i.e. the model is able
    to see the bug the early flush fixes."""
    pages = [4] + [2] * 400
    orig = Warp.block_setup

    def no_early_flush(self, first_tile):
        cp, end = self.cp, self.cp_end_g
        self.cp = -1            # hide the page from the early-flush test ...
        orig(self, first_tile)
        self.cp = cp            # ... and restore it (extent bookkeeping as in the kernel before the fix)
        if cp >= 0 and end < 0 and self.cmask:
            self.cp_end_g = self.g_base + (self.cmask & -self.cmask).bit_length() - 1

    Warp.block_setup = no_early_flush
    try:
        with pytest.raises(AssertionError):
            run_model(pages, 2, 0)
    finally:
        Warp.block_setup = orig
