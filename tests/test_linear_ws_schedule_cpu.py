"""Host model of the barrier schedule of linear_ws_kernel (csrc/fp_linear.cu), the weight-stationary K = 512 linear
kernel: one producer thread and two consumer warpgroups that take alternate 64-row tiles of a CTA's range.

The model runs the kernel's program order for each role over the same mbarriers (parity waits with the hardware's
rule: a wait on parity P returns once the barrier's current phase has the other parity), named barriers and TMA
transfers, which complete at arbitrary later points.  A random scheduler interleaves the roles and the transfers.  The
test asserts, for every distinct range shape a launch gives its CTAs, that:

  * no wait blocks forever (every role finishes);
  * every stage, the weight panel and the staging slabs hold the data the reader expects when it reads them, and no
    transfer writes a buffer while a reader still holds it;
  * every fill of a ring stage is released exactly once, by the warpgroup that read it.
"""
import random

import pytest

K_BLOCKS = 8  # the ring holds one tile: stage kb = k-block kb
ROWS = 64
COLS = 128
SMS = 132


class Barrier:
    def __init__(self, count):
        self.count, self.arrived, self.tx, self.phases = count, 0, 0, 0

    def arrive(self, n=1):
        self.arrived += n
        assert self.arrived <= self.count, "more arrivals than the barrier's count in one phase"
        self._complete()

    def expect_tx(self, units):
        self.tx += units
        self.arrive()

    def complete_tx(self):
        self.tx -= 1
        assert self.tx >= 0
        self._complete()

    def _complete(self):
        if self.arrived == self.count and self.tx == 0:
            self.arrived = 0
            self.phases += 1

    def try_wait(self, parity):
        return (self.phases & 1) != parity


class NamedBarrier:
    """bar.sync / bar.arrive over 256 threads: two warpgroups, counted as 1 each here"""

    def __init__(self):
        self.arrived, self.generation = 0, 0

    def arrive(self):
        self.arrived += 1
        assert self.arrived <= 2, "a named barrier received a third arrival in one generation"
        if self.arrived == 2:
            self.arrived = 0
            self.generation += 1


class Cta:
    def __init__(self, n, jb, rows_per_panel, i0, has_res, rng):
        self.n, self.jb, self.R, self.i0, self.has_res, self.rng = n, jb, rows_per_panel, i0, has_res, rng
        self.reload = jb < n
        self.full = [Barrier(1) for _ in range(K_BLOCKS)]
        self.empty = [Barrier(1) for _ in range(K_BLOCKS)]  # one warpgroup (128 threads) releases a fill
        self.panel_full, self.panel_empty = Barrier(1), Barrier(2)
        self.res_full = [Barrier(1), Barrier(1)]
        self.order = [NamedBarrier(), NamedBarrier()]
        self.stage = [None] * K_BLOCKS   # item whose k-block the stage holds
        self.stage_holder = [None] * K_BLOCKS
        self.panel = None
        self.panel_holders = set()
        self.slabs = [None, None]        # per warpgroup: ("res" | "out", item)
        self.stores = [[], []]           # per warpgroup: outstanding TMA stores (read the slabs)
        self.res_in_flight = [0, 0]
        self.fills = [0] * K_BLOCKS
        self.releases = {}
        self.transfers = []              # pending TMA transfers: callables

    def panel_of(self, j):
        return (self.i0 + j) // self.R

    # ---- TMA transfers
    def load_panel(self, pn):
        assert not self.panel_holders, "the panel is overwritten while a warpgroup reads it"

        def done():
            assert not self.panel_holders
            self.panel = pn
            self.panel_full.complete_tx()
        self.transfers.append(done)

    def load_stage(self, kb, item):
        assert self.stage_holder[kb] is None, "a stage is overwritten while a warpgroup reads it"
        self.fills[kb] += 1

        def done():
            assert self.stage_holder[kb] is None
            self.stage[kb] = item
            self.full[kb].complete_tx()
        self.transfers.append(done)

    def load_res(self, w, item):
        assert not self.stores[w], "the residual lands in slabs a store still reads"
        self.res_in_flight[w] += 1

        def done():
            assert not self.stores[w]
            self.slabs[w] = ("res", item)
            self.res_in_flight[w] -= 1
            self.res_full[w].complete_tx()
        self.transfers.append(done)

    def store(self, w, item):
        tok = object()
        self.stores[w].append(tok)

        def done():
            assert self.slabs[w] == ("out", item), "the slabs changed under a store"
            self.stores[w].remove(tok)
        self.transfers.append(done)

    # ---- roles, in the kernel's program order; each yield is a wait predicate
    def producer(self):
        for j in range(self.n):
            if j == self.jb:
                yield lambda: self.panel_empty.try_wait(0)
                self.panel_full.expect_tx(1)
                self.load_panel(self.panel_of(0) + 1)
            for kb in range(K_BLOCKS):
                yield lambda kb=kb, j=j: self.empty[kb].try_wait((j & 1) ^ 1)
                self.full[kb].expect_tx(1)
                self.load_stage(kb, self.i0 + j)

    def consumer(self, w):
        if self.reload and w >= self.jb:
            self.panel_empty.arrive()
        it = 0
        for j in range(w, self.n, 2):
            item = self.i0 + j
            pn = self.panel_of(j)
            if j > 0:
                bar = self.order[w]
                gen = bar.generation
                bar.arrive()
                yield lambda bar=bar, gen=gen: bar.generation > gen
            yield lambda j=j: self.panel_full.try_wait(1 if j >= self.jb else 0)
            assert self.panel == pn, f"warpgroup {w} tile {j}: panel {self.panel}, expected {pn}"
            self.panel_holders.add(w)
            for kb in range(K_BLOCKS):
                yield lambda kb=kb, j=j: self.full[kb].try_wait(j & 1)
                assert self.stage[kb] == item, f"warpgroup {w} tile {j} k-block {kb}: stage holds {self.stage[kb]}"
                assert self.stage_holder[kb] is None
                self.stage_holder[kb] = w
                if kb == 0:
                    yield lambda: not self.stores[w]  # the leader's cp.async.bulk.wait_group.read 0
                    if self.has_res:
                        self.res_full[w].expect_tx(1)
                        self.load_res(w, item)
                if kb > 0:
                    self.release(w, kb - 1, item)
            if j + 1 < self.n:
                self.order[w ^ 1].arrive()
            self.release(w, K_BLOCKS - 1, item)
            self.panel_holders.discard(w)
            if self.reload and j < self.jb <= j + 2:
                self.panel_empty.arrive()
            if self.has_res:
                yield lambda it=it: self.res_full[w].try_wait(it & 1)
                assert self.slabs[w] == ("res", item), f"warpgroup {w} tile {j}: slabs hold {self.slabs[w]}"
            assert not self.stores[w] and not self.res_in_flight[w]
            self.slabs[w] = ("out", item)
            self.store(w, item)
            it += 1
        yield lambda: not self.stores[w]

    def release(self, w, kb, item):
        assert self.stage_holder[kb] == w and self.stage[kb] == item
        self.stage_holder[kb] = None
        key = (kb, self.fills[kb])
        assert key not in self.releases, f"stage {kb} fill {self.fills[kb]} released twice"
        self.releases[key] = w
        self.empty[kb].arrive()

    def run(self):
        # thread 0 issues the first panel ahead of the CTA-wide barrier that releases the roles
        self.panel_full.expect_tx(1)
        self.load_panel(self.panel_of(0))
        roles = {"producer": self.producer(), "wg0": self.consumer(0), "wg1": self.consumer(1)}
        waits = {}
        for name, g in list(roles.items()):
            try:
                waits[name] = next(g)
            except StopIteration:
                del roles[name]
        while roles or self.transfers:
            ready = [name for name in roles if waits[name]()]
            choices = [("role", name) for name in ready] + [("tma", i) for i in range(len(self.transfers))]
            assert choices, f"deadlock: {sorted(roles)} wait forever (n={self.n}, jb={self.jb})"
            kind, x = self.rng.choice(choices)
            if kind == "tma":
                self.transfers.pop(x)()
                continue
            try:
                waits[x] = next(roles[x])
            except StopIteration:
                del roles[x]
        # every fill was read and released once
        for kb in range(K_BLOCKS):
            assert self.fills[kb] == self.n
            assert sorted(f for (s, f) in self.releases if s == kb) == list(range(1, self.n + 1))
        assert self.panel_full.phases == (2 if self.reload else 1)


def range_shapes(M, Cout, grid=None):
    """(n, jb, i0) of every CTA of a launch, as linear_ws_kernel splits the items, with duplicates of (n, jb) dropped"""
    R = -(-M // ROWS)
    total = (Cout // COLS) * R
    grid = grid or min(SMS, total)
    shapes = {}
    for b in range(grid):
        i0 = b * total // grid
        n = (b + 1) * total // grid - i0
        panel0 = i0 // R
        jb = min(n, (panel0 + 1) * R - i0)
        assert (i0 + n - 1) // R <= panel0 + 1, "a range crosses more than one panel boundary"
        shapes.setdefault((n, jb), i0)
    return R, [(n, jb, i0) for (n, jb), i0 in shapes.items()]


@pytest.mark.parametrize("M", [100800, 99600, 12800, 400])
@pytest.mark.parametrize("Cout", [512, 1536, 3072])
@pytest.mark.parametrize("has_res", [False, True])
def test_schedule_completes_and_reads_what_was_loaded(M, Cout, has_res):
    R, shapes = range_shapes(M, Cout)
    assert shapes
    for n, jb, i0 in shapes:
        Cta(n, jb, R, i0, has_res, random.Random(hash((M, Cout, has_res, n, jb)) & 0xFFFF)).run()


@pytest.mark.parametrize("n,jb", [(1, 1), (2, 1), (3, 1), (3, 2), (5, 4), (6, 3), (7, 1), (9, 8), (12, 6), (48, 17)])
@pytest.mark.parametrize("has_res", [False, True])
def test_panel_boundary_inside_the_range(n, jb, has_res):
    """Ranges whose boundary follows the first tile (warpgroup 1 never reads the first panel), falls on either
    warpgroup's tile, or precedes the last tile; many interleavings each."""
    R = 64
    i0 = R - jb  # the range's first jb tiles are the end of panel 0
    for seed in range(20):
        Cta(n, jb, R, i0, has_res, random.Random(seed)).run()


def test_the_model_sees_a_missing_order_barrier():
    """Without the ordering of the k-loops a warpgroup can pass a parity wait on the fill two tiles back."""

    found = False
    for seed in range(200):
        c = Cta(6, 6, 64, 0, False, random.Random(seed))
        c.order = [_Open(), _Open()]
        try:
            c.run()
        except AssertionError:
            found = True
            break
    assert found


class _Open(NamedBarrier):
    """a named barrier that never blocks"""

    def arrive(self):
        self.generation += 1
