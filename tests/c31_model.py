"""CPU model of the barrier protocol of conv_c31_kernel (deep-image-retrieval_b200/csrc/conv_c31.cuh, protocols 1-4).

Two consumer warpgroups run their programs; TMA loads, TMA store reads and the weight refills complete as separate
events, and a seeded scheduler interleaves all of them at random.  The model tracks what each ring slot, staging
buffer and T2 buffer holds and who still reads it, and reports:
  "ok"                          both programs finished and every read saw the data it expects;
  "deadlock"                    nothing can run and a program has not finished;
  "expected ... got ..."        a warpgroup read a slot or buffer that holds other data (a stale or early fill);
  "race ..."                    a TMA load was issued into a buffer that a store or an MMA still reads.
mbarrier waits are parity waits, as on the device: try_wait.parity(P) passes once the barrier's completed-phase count
has a parity other than P.  wgmma reads of the ring are complete at the next wait_group, so a slot is read when the
warpgroup consumes it and released one group later; conv1's reads of a staging buffer last until the next wait_group 0.

Switches reproduce the mistakes the protocol rules out:
  empty_count=1        one arrival per empty barrier instead of one per warpgroup;
  skip_wait_read=True  a residual load without waiting for the previous stores to have read the buffer;
  early_res=True       the next residual load issued before the wait_group 0 that ends the previous conv1's reads.
"""
import random
from dataclasses import dataclass


@dataclass(frozen=True)
class Config:
    stages: int
    kb: int          # conv3 K blocks (Cm / 64)
    ns: int          # 64-channel blocks per chunk (conv1 K steps per chunk)
    nh1: int         # conv1 wgmmas per K step
    nc: int          # chunks per tile
    nbuf: int        # staging buffers
    tiles: int       # tiles of this CTA
    empty_count: int = 2
    skip_wait_read: bool = False
    early_res: bool = False


def kernel_config(cm, tiles, stages=None, **bugs):
    """The kernel's constants at Cm = 64 / 128 / 256 (C31Smem)."""
    n3, nb1 = 128, min(cm, 128)
    st = {64: 8, 128: 8, 256: 6}[cm] if stages is None else stages
    return Config(st, cm // 64, n3 // 64, cm // nb1, 4 * cm // n3, 256 // n3, tiles, **bugs)


class Fail(Exception):
    pass


class Barrier:
    def __init__(self, count):
        self.count, self.arrived, self.done = count, 0, 0

    def arrive(self):
        self.arrived += 1
        if self.arrived == self.count:
            self.arrived = 0
            self.done += 1

    def passed(self, parity):
        return (self.done & 1) != parity


class Buffer:
    def __init__(self):
        self.data = None
        self.readers = set()

    def load(self, what, sim, bar):
        if self.readers:
            raise Fail("race: load of %s into a buffer still read by %s" % (what, sorted(self.readers)))
        self.readers.add("incoming")          # a landing load is a write in flight: writing over it is a race too
        sim.events.append((self, what, bar))

    def write(self, what):
        if self.readers:
            raise Fail("race: epilogue writes %s while %s read the buffer" % (what, sorted(self.readers)))
        self.data = what

    def expect(self, what):
        if self.data != what:
            raise Fail("expected %s got %s" % (what, self.data))


class Sim:
    def __init__(self, cfg, seed):
        self.cfg, self.rng = cfg, random.Random(seed)
        s = cfg.stages
        self.full = [Barrier(1) for _ in range(s)]
        self.empty = [Barrier(cfg.empty_count) for _ in range(s)]
        self.slot = [None] * s
        self.events = []             # (target, value, barrier): a TMA load that lands when the scheduler picks it
        self.stores = []             # (warpgroup, buffers, id): bulk groups whose smem reads are in flight
        self.fills = cfg.tiles * cfg.nc * (cfg.kb + cfg.ns * cfg.nh1)

    def fill(self, f):
        """Warpgroup 0's leader loads fill f once both warpgroups have released the slot's previous fill."""
        if f >= self.fills:
            return
        s = f % self.cfg.stages
        while not self.empty[s].passed(((f // self.cfg.stages) & 1) ^ 1):
            yield
        self.events.append((("slot", s), f, self.full[s]))


def warpgroup(sim, w):
    cfg, S = sim.cfg, sim.cfg.stages
    t2 = Buffer()
    stg = [Buffer() for _ in range(cfg.nbuf)]
    t2_bar = Barrier(1)
    res_bar = [Barrier(1) for _ in range(cfg.nbuf)]
    groups = []                      # this warpgroup's bulk groups, oldest first: sets of buffers still being read
    g = 0
    held = None
    conv1_reading = []

    def release(f):
        sim.empty[f % S].arrive()
        if w == 0:
            yield from sim.fill(f + S)

    def consume(expect_fill):
        nonlocal g, held
        s = g % S
        while not sim.full[s].passed((g // S) & 1):
            yield
        if sim.slot[s] != expect_fill:
            raise Fail("expected fill %d in slot %d got %s" % (expect_fill, s, sim.slot[s]))
        if held is not None:
            yield from release(held)
        held = g
        g += 1

    def wait0():
        nonlocal held
        for b in conv1_reading:
            stg[b].readers.discard("conv1")
        conv1_reading.clear()
        if held is not None:
            yield from release(held)
        held = None

    def wait_read(n):          # cp.async.bulk.wait_group.read n: every group but the n most recent has read smem
        while any(x["reading"] for x in groups[:len(groups) - n]):
            yield

    def store(bufs):
        grp = {"reading": True, "bufs": bufs}
        for b in bufs:
            stg[b].readers.add("store%d" % id(grp))
        groups.append(grp)
        sim.stores.append((grp, [stg[b] for b in bufs]))

    def load_res(tile, c):
        b = c % cfg.nbuf
        stg[b].load(("res", tile, c), sim, res_bar[b])

    if w == 0:
        for f in range(S):
            yield from sim.fill(f)
    t2.load(("t2", 0), sim, t2_bar)
    load_res(0, 0)
    q = 0
    per_chunk = cfg.kb + cfg.ns * cfg.nh1
    for i in range(cfg.tiles):
        while not t2_bar.passed(i & 1):
            yield
        t2.expect(("t2", i))
        for c in range(cfg.nc):
            b = c % cfg.nbuf
            base = (i * cfg.nc + c) * per_chunk
            if cfg.early_res and c + 1 < cfg.nc:
                yield from wait_read(0)
                load_res(i, c + 1)
            t2.readers.add("conv3")
            for kc in range(cfg.kb):
                yield from consume(base + kc)
            t2.readers.discard("conv3")
            yield from wait0()
            while not res_bar[b].passed((q // cfg.nbuf) & 1):
                yield
            stg[b].readers.discard("incoming")
            stg[b].expect(("res", i, c))
            stg[b].write(("x", i, c))
            yield
            store([b])
            if c + 1 < cfg.nc:
                if not cfg.early_res:
                    if not cfg.skip_wait_read:
                        yield from wait_read(1)
                    load_res(i, c + 1)
            elif i + 1 < cfg.tiles:
                t2.load(("t2", i + 1), sim, t2_bar)
            stg[b].readers.add("conv1")
            conv1_reading.append(b)
            for e in range(cfg.ns * cfg.nh1):
                yield from consume(base + cfg.kb + e)
            q += 1
        yield from wait0()
        yield from wait_read(0)
        for b in range(cfg.nbuf):
            stg[b].write(("t1", i))
        yield
        store(list(range(cfg.nbuf)))
        if i + 1 < cfg.tiles:
            yield from wait_read(0)
            load_res(i + 1, 0)


def simulate(cfg, seed, max_steps=200000):
    sim = Sim(cfg, seed)
    progs = [warpgroup(sim, 0), warpgroup(sim, 1)]
    alive = [True, True]
    try:
        for _ in range(max_steps):
            choices = [("wg", w) for w in range(2) if alive[w]]
            choices += [("event", k) for k in range(len(sim.events))]
            choices += [("store", k) for k in range(len(sim.stores))]
            if not any(alive) and not sim.events:
                return "ok"
            kind, k = sim.rng.choice(choices)
            if kind == "wg":
                try:
                    next(progs[k])
                except StopIteration:
                    alive[k] = False
            elif kind == "event":
                target, value, bar = sim.events.pop(k)
                if isinstance(target, tuple):
                    sim.slot[target[1]] = value
                else:
                    target.data = value
                    target.readers.discard("incoming")
                bar.arrive()
            elif kind == "store":
                grp, bufs = sim.stores.pop(k)
                grp["reading"] = False
                for buf in bufs:
                    buf.readers.discard("store%d" % id(grp))
            if not any(alive) and not sim.events:
                return "ok"
        return "deadlock"
    except Fail as e:
        return str(e)
