"""The schedule of tensor_scan_s8_kernel (csrc/tensor_scan.cu) stepped on the CPU: one TMA producer, two consumer
warpgroups that take turns at the tensor pipe through two named barriers, a ring of mbarrier-guarded stages and the
resident query tile's barrier.  Every interleaving the model draws must run to the end (no deadlock), no wait may be
satisfied by a phase other than the one it is meant for (parity aliasing), no named barrier may complete without its
waiting warpgroup, and every barrier must be balanced when the CTA ends.  This is a model of the kernel's protocol,
written from the same formulas; it runs no device code.
"""
import random

import pytest


class MBar:
    """mbarrier: `count` arrivals complete a phase; `done` = completed phases"""

    def __init__(self, count):
        self.count, self.pending, self.done = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.done += 1
            self.pending = self.count

    def passes(self, parity):   # mbarrier.try_wait.parity: the phase of that parity has completed
        return (self.done & 1) != parity


class NamedBar:
    """bar.sync / bar.arrive over 256 threads: each warpgroup contributes 128"""

    def __init__(self):
        self.arrived, self.waiter, self.released = 0, None, 0

    def _add(self):
        self.arrived += 128
        if self.arrived == 256:
            assert self.waiter is not None, "a named barrier completed without its waiting warpgroup"
            self.arrived, self.waiter, self.released = 0, None, self.released + 1

    def arrive(self, who):
        assert self.waiter != who
        self._add()

    def sync(self, who):   # returns the generation to wait for
        assert self.waiter is None
        gen = self.released
        self.waiter = who
        self._add()
        return gen


def cta_tiles(ntiles, G, g):
    return (ntiles - g + G - 1) // G if g < ntiles else 0


def run(ntiles, G, g, stages, kblocks, n_rows, seed):
    T = cta_tiles(ntiles, G, g)
    full = [MBar(1) for _ in range(stages)]
    empty = [MBar(4) for _ in range(stages)]
    qbar = MBar(1)
    turn = [NamedBar(), NamedBar()]   # TS8_BAR_TURN + w: "warpgroup w may issue its K loop"
    loaded = {}                       # ring position -> (tile, half, kb) the producer put there

    def wait(pred):
        while not pred():
            yield

    def producer():
        if T == 0:
            return
        qbar.arrive()                 # expect_tx + the query tile's loads (complete_tx modelled as immediate)
        s = phase = 0
        p = 0
        for t in range(T):
            nt = g + t * G
            for h in range(2):
                hrow0 = nt * 256 + h * 128
                for kb in range(kblocks):
                    yield from wait(lambda: empty[s].passes(phase ^ 1))
                    assert empty[s].done == p // stages, "producer passed an empty barrier of another phase"
                    loaded[p] = (t, h, kb, hrow0 < n_rows)
                    full[s].arrive()  # live half: expect_tx + TMA (completes later, modelled at once); dead: plain arrive
                    p += 1
                    s += 1
                    if s == stages:
                        s, phase = 0, phase ^ 1

    def consumer(wg):
        if T == 0:
            return
        if wg == 1:
            turn[0].arrive(1)         # warpgroup 0 takes the first turn
        yield from wait(lambda: qbar.passes(0))
        for t in range(T):
            p0 = (2 * t + wg) * kblocks
            s, phase = p0 % stages, (p0 // stages) & 1
            gen = turn[wg].sync(wg)
            yield from wait(lambda: turn[wg].released > gen)
            prev = None
            for kb in range(kblocks):
                p = p0 + kb
                yield from wait(lambda: full[s].passes(phase))
                assert full[s].done == p // stages + 1, "consumer passed a full barrier of another phase"
                assert loaded[p][:3] == (t, wg, kb), ("stage holds the wrong k-block", loaded[p], (t, wg, kb))
                if kb > 0:
                    for _ in range(4):
                        empty[prev].arrive()
                prev = s
                s += 1
                if s == stages:
                    s, phase = 0, phase ^ 1
                yield
            if wg == 0:
                turn[1].arrive(0)
            elif t + 1 < T:
                turn[0].arrive(1)
            if kblocks > 0:
                for _ in range(4):
                    empty[prev].arrive()
            yield                      # epilogue and refresh

    rng = random.Random(seed)
    agents = {"producer": producer(), "wg0": consumer(0), "wg1": consumer(1)}
    live = dict(agents)
    stalled = 0
    while live:
        name = rng.choice(sorted(live))
        try:
            before = (sum(m.done for m in full + empty), turn[0].released, turn[1].released, len(loaded))
            next(live[name])
            after = (sum(m.done for m in full + empty), turn[0].released, turn[1].released, len(loaded))
            stalled = 0 if after != before else stalled + 1
        except StopIteration:
            del live[name]
            stalled = 0
        assert stalled < 10_000, f"deadlock: {sorted(live)} blocked (T={T})"
    for b in turn:
        assert b.arrived == 0 and b.waiter is None, "named barrier left with pending arrivals"
    assert len(loaded) == 2 * T * kblocks
    for m in full:
        assert m.pending == m.count
    for m in empty:
        assert m.pending == m.count
    if T:
        assert sum(m.done for m in full) == 2 * T * kblocks == sum(m.done for m in empty)
    return T


CASES = [
    # ntiles, G, g, stages, kblocks, n_rows
    (1, 1, 0, 6, 6, 100),          # one tile whose upper half lies wholly past the corpus end
    (1, 1, 0, 6, 6, 256),
    (3, 1, 0, 6, 6, 3 * 256 - 5),  # odd tile count, partial last tile
    (7, 2, 1, 6, 6, 7 * 256 - 130),
    (5, 8, 3, 6, 6, 5 * 256),      # ntiles < G, a CTA with one tile
    (5, 8, 6, 6, 6, 5 * 256),      # ntiles < G, a CTA with none
    (9, 4, 0, 4, 8, 9 * 256 - 200),
    (11, 3, 2, 5, 2, 11 * 256),    # more stages than one turn's k-blocks
    (10, 2, 0, 4, 4, 10 * 256 - 128),
    (6, 1, 0, 4, 1, 6 * 256 - 1),
    (2441, 8, 7, 6, 6, 10_000_000),  # the headline: 10M rows, 8 CTA groups
]


@pytest.mark.parametrize("case", CASES)
def test_schedule_never_deadlocks(case):
    ntiles, G, g, stages, kblocks, n_rows = case
    for seed in range(20 if ntiles < 100 else 2):
        run(ntiles, G, g, stages, kblocks, n_rows, seed)


def test_schedule_sweep():
    rng = random.Random(7)
    for _ in range(300):
        ntiles = rng.randint(0, 20)
        G = rng.randint(1, 9)
        g = rng.randint(0, G - 1)
        stages = rng.randint(4, 6)
        kblocks = rng.randint(1, 8)
        n_rows = max(0, ntiles * 256 - rng.randint(0, 255)) if ntiles else 0
        run(ntiles, G, g, stages, kblocks, n_rows, rng.randint(0, 1 << 30))
