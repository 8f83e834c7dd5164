"""A CPU model of the ping-pong consumer protocol of conv_pers_kernel (csrc/conv_pers.cuh, PP = true).

One TMA producer fills a STAGES-deep operand ring (and, for HALO launches, an NP-deep patch ring) in tile order; two
consumer warpgroups take the CTA-local tiles alternately (tile i -> warpgroup i & 1).  Each consumer warpgroup is four
warps, and every warp is an agent of its own: a generator that yields one atomic step at a time.  A step that waits is
resumed only once its condition holds; an mbarrier wait uses the hardware's `try_wait.parity` semantics - it passes iff
the barrier's current phase parity differs from the one asked for, so a waiter two phases behind or ahead passes on the
wrong phase or never passes.  What couples the warps of a warpgroup is modelled as the hardware provides it:
- a wgmma group completes once all four warps have issued it (`wgmma.wait_group` waits for that);
- the epilogue's 128-thread named barrier;
- everything else (mbarrier waits, the mma_done arrival) is per warp.
Warp 0 of a warpgroup is its leader: it hands ring / patch slots back, loads the residual and stores the output.  TMA
loads and stores are agents too, so they land and read in any order.  A random scheduler with a random speed per
agent interleaves everything, so some warps lag far behind their siblings.

The model records what each warp reads: every ring / patch slot must hold the fill it expects (fill index
g = i * k_iters + it, patch index gp = i * cin_blocks + kc) when the warp issues its wgmma on it, and every staging
buffer must hold the residual of its own tile and be stored from the epilogue of its own tile.  A state in which no agent
can move before all have finished is a deadlock.

Switches reproduce the bugs the kernel's invariants rule out: `order=False` drops the mma_done handover,
`handover_warps=1` lets only the leader warp arrive on mma_done (count 1), `empty_count=2` expects two arrivals per fill
(the cooperative count), `shared_staging=True` gives both warpgroups one set of staging buffers and one residual barrier.
"""
import random
from dataclasses import dataclass

WARPS = 4


class Violation(Exception):
    pass


class MBarrier:
    """mbarrier: an arrival count and a transaction count per phase; `phase` counts completed phases."""

    def __init__(self, count):
        self.count = count
        self.pending = count
        self.tx = 0
        self.phase = 0

    def _complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        self.pending -= 1
        self._complete()

    def arrive_expect_tx(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._complete()

    def try_wait(self, parity):
        return (self.phase & 1) != parity


@dataclass
class Config:
    stages: int
    k_iters: int             # k-iterations per tile (HALO: 9 * cin_blocks)
    tiles: int               # CTA-local tiles
    halo: bool = False
    np_slots: int = 2        # patch ring depth (HALO)
    has_res: bool = True
    order: bool = True       # mma_done handover (invariant 1)
    handover_warps: int = WARPS    # warps arriving on mma_done per tile (the barrier's count)
    empty_count: int = 1     # arrivals expected per fill on the empty barriers (invariant 3)
    shared_staging: bool = False   # one staging set / residual barrier for both warpgroups (breaks invariant 4)

    @property
    def cin_blocks(self):
        return self.k_iters // 9 if self.halo else 1


def _wait(bar, parity):
    return ("until", lambda: bar.try_wait(parity))


class Sim:
    def __init__(self, cfg: Config, seed: int):
        self.cfg = cfg
        self.rng = random.Random(seed)
        S, NP = cfg.stages, cfg.np_slots
        self.full = [MBarrier(1) for _ in range(S)]
        self.empty = [MBarrier(cfg.empty_count) for _ in range(S)]
        self.pfull = [MBarrier(1) for _ in range(NP)]
        self.pempty = [MBarrier(cfg.empty_count) for _ in range(NP)]
        nstg = 1 if cfg.shared_staging else 2
        self.res_bar = [MBarrier(1) for _ in range(nstg)]
        self.mma_done = [MBarrier(cfg.handover_warps), MBarrier(cfg.handover_warps)]
        self.ring = [None] * S                  # fill index held by each operand slot
        self.patch = [None] * NP                # patch index held by each patch slot
        self.stg = [[None] * WARPS for _ in range(nstg)]   # per staging set, the rows of each warp: ('res' | 'out', tile)
        self.stores_in_flight = [0, 0]          # TMA stores of each warpgroup leader not yet done reading
        self.issued = [[0] * WARPS for _ in range(2)]      # wgmma groups issued by each warp
        self.named = [[0] * WARPS for _ in range(2)]       # named-barrier syncs reached by each warp
        self.agents = []
        self.reads = []                         # (warpgroup, warp, 'ring' | 'patch', index)

    # ------------------------------------------------------------------ asynchronous copies
    def _spawn(self, gen):
        self.agents.append([gen, None, 2.0 ** self.rng.uniform(-5, 0)])   # generator, pending request, speed

    def _land_ring(self, s, g):
        yield None
        self.ring[s] = g
        self.full[s].complete_tx(1)

    def _land_patch(self, ps, gp):
        yield None
        self.patch[ps] = gp
        self.pfull[ps].complete_tx(1)

    def _land_res(self, w, tile):
        yield None
        self.stg[w] = [("res", tile)] * WARPS
        self.res_bar[w].complete_tx(1)

    def _store(self, wg, w, tile):
        yield None
        if self.stg[w] != [("out", tile)] * WARPS:
            raise Violation("warpgroup %d stored staging %s for tile %d" % (wg, self.stg[w], tile))
        self.stores_in_flight[wg] -= 1

    # ------------------------------------------------------------------ producer (unchanged by the ping-pong mode)
    def producer(self):
        c, S, NP = self.cfg, self.cfg.stages, self.cfg.np_slots
        g = gp = 0
        for _ in range(c.tiles):
            for kc in range(c.cin_blocks if c.halo else 1):
                if c.halo:
                    ps = gp % NP
                    yield _wait(self.pempty[ps], ((gp // NP) & 1) ^ 1)
                    self.pfull[ps].arrive_expect_tx(1)
                    self._spawn(self._land_patch(ps, gp))
                    gp += 1
                for _it in range(9 if c.halo else c.k_iters):
                    s = g % S
                    yield _wait(self.empty[s], ((g // S) & 1) ^ 1)
                    self.full[s].arrive_expect_tx(1)
                    self._spawn(self._land_ring(s, g))
                    g += 1

    # ------------------------------------------------------------------ one warp of consumer warpgroup wg
    def _check(self, wg, wp, kind, slot, want):
        have = (self.ring if kind == "ring" else self.patch)[slot]
        if have != want:
            raise Violation("warpgroup %d warp %d read %s slot %d holding %s, expected %s" % (wg, wp, kind, slot, have, want))

    def _named_sync(self, wg, wp):
        self.named[wg][wp] += 1
        n = self.named[wg][wp]
        return ("until", lambda: min(self.named[wg]) >= n)

    def consumer_warp(self, wg, wp):
        c, S, NP = self.cfg, self.cfg.stages, self.cfg.np_slots
        w = 0 if c.shared_staging else wg
        leader = wp == 0
        issued = self.issued[wg]

        def wgmma_wait(n):
            """wgmma.wait_group n: all but this warp's n most recent groups are complete, i.e. issued by all warps."""
            mine = issued[wp]
            return ("until", lambda: min(issued) >= mine - n)

        def issue(kind, slot, want, index, record=True):
            self._check(wg, wp, kind, slot, want)
            if record:
                self.reads.append((wg, wp, kind, index))

        for i in range(wg, c.tiles, 2):
            j = i >> 1
            if c.has_res and leader:
                # its own earlier stores have finished reading the staging set, then the residual load
                while self.stores_in_flight[wg]:
                    yield ("spin",)
                self.res_bar[w].arrive_expect_tx(1)
                self._spawn(self._land_res(w, i))
            g = i * c.k_iters                                       # invariant 2
            gp = i * c.cin_blocks
            if c.order and i > 0:
                yield _wait(self.mma_done[wg ^ 1], ((i - 1) >> 1) & 1)   # invariant 1
            prev_last = False
            for kc in range(c.cin_blocks if c.halo else 1):
                if c.halo:
                    ps = gp % NP
                    yield _wait(self.pfull[ps], (gp // NP) & 1)
                for tap in range(9 if c.halo else c.k_iters):
                    s = g % S
                    yield _wait(self.full[s], (g // S) & 1)
                    issue("ring", s, g, g)
                    if c.halo:                                      # every tap reads the patch
                        issue("patch", gp % NP, gp, gp, record=tap == 0)
                    issued[wp] += 1                                 # wgmma + commit
                    yield wgmma_wait(1)                             # the previous group is done
                    if leader and (kc or tap):
                        self.empty[(g - 1) % S].arrive()
                        if prev_last:
                            self.pempty[(gp - 1) % NP].arrive()
                    prev_last = c.halo and tap == 8
                    g += 1
                gp += 1 if c.halo else 0
            if c.order and wp < c.handover_warps:
                self.mma_done[wg].arrive()                          # this warp has passed every full-barrier wait
            yield wgmma_wait(0)
            if leader:
                self.empty[(g - 1) % S].arrive()
                if c.halo:
                    self.pempty[(gp - 1) % NP].arrive()
            # epilogue
            if c.has_res:
                yield _wait(self.res_bar[w], j & 1)
                if self.stg[w][wp] != ("res", i):
                    raise Violation("warpgroup %d warp %d epilogue of tile %d found staging %s" % (wg, wp, i, self.stg[w][wp]))
            else:
                while leader and self.stores_in_flight[wg]:
                    yield ("spin",)
                yield self._named_sync(wg, wp)
            self.stg[w][wp] = ("out", i)
            yield self._named_sync(wg, wp)
            if leader:
                self.stores_in_flight[wg] += 1
                self._spawn(self._store(wg, w, i))

    # ------------------------------------------------------------------ scheduler
    def run(self, max_steps=200_000):
        """-> 'ok', 'deadlock' or the text of the first violation."""
        self._spawn(self.producer())
        for wg in (0, 1):
            for wp in range(WARPS):
                self._spawn(self.consumer_warp(wg, wp))
        steps = 0
        try:
            while self.agents:
                ready = [a for a in self.agents if self._ready(a)]
                if not ready:
                    return "deadlock"
                a = self.rng.choices(ready, weights=[r[2] for r in ready])[0]
                try:
                    a[1] = next(a[0])
                except StopIteration:
                    self.agents.remove(a)
                steps += 1
                if steps > max_steps:
                    return "deadlock"
        except Violation as e:
            return str(e)
        return "ok"

    @staticmethod
    def _ready(a):
        req = a[1]
        if req is None or req[0] == "spin":    # "spin" re-checks its condition when scheduled
            return True
        return req[1]()


def expected_reads(cfg: Config):
    """Every (warpgroup, warp, kind, index) a correct run reads, in no particular order."""
    out = []
    for i in range(cfg.tiles):
        wg = i & 1
        for wp in range(WARPS):
            if cfg.halo:
                out += [(wg, wp, "patch", i * cfg.cin_blocks + kc) for kc in range(cfg.cin_blocks)]
            out += [(wg, wp, "ring", i * cfg.k_iters + it) for it in range(cfg.k_iters)]
    return sorted(out)


def simulate(cfg: Config, seed: int):
    """One random interleaving: 'ok' only if it finished and read exactly the expected fills."""
    sim = Sim(cfg, seed)
    res = sim.run()
    if res == "ok" and sorted(sim.reads) != expected_reads(cfg):
        return "reads differ from the expected fills"
    return res
