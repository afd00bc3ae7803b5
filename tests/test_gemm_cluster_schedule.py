"""CPU: a model of the barrier protocol of the 2-CTA cluster GEMM (`gemm_bf16_tn_kernel<..., CLUSTER = 2>`).

Each CTA of a cluster has one TMA producer and two ping-pong consumer warpgroups that walk the ring with the kernel's
cursor rules (`StageRing` advance / skip, the two order barriers, the persistent unit loop).  A producer loads its own
A tile and multicasts its half of the shared W tile into the same stage of both CTAs; the empty barriers count the
consumer warps of both CTAs.  The model runs the agents under many random interleavings, with the TMA copies landing
at random later moments, and checks that

* every wait completes (no deadlock) and a CTA exits only when nothing can still land on it or arrive on its barriers;
* every parity wait is at most one phase ahead of its barrier (otherwise the parity would alias and pass early);
* a stage is written only after the consumers of the receiving CTA have released its previous contents;
* both CTAs issue the same number of multicasts into every stage;
* every output tile is computed exactly once, and a phantom tile (odd tiles_m) only past the last m-tile.

It is a rehearsal of the protocol, not of the arithmetic: a wedged pipeline on the GPU is a trap."""
import random

import pytest

STAGES = 6            # GemmCfg<128>::STAGES
A_BYTES = 128 * 64 * 2
W_BYTES = 128 * 64 * 2
GM = 8                # gemm_tile_coords band height


def tile_coords(tile, tiles_m, tiles_n):
    per_group = GM * tiles_n
    g = tile // per_group
    first_m = g * GM
    gsize = min(GM, tiles_m - first_m)
    within = tile - g * per_group
    return first_m + within % gsize, within // gsize


class Bar:
    """mbarrier: `count` arrivals plus a transaction byte count per phase; `done` = completed phases."""

    def __init__(self, count):
        self.count, self.pending, self.tx, self.done = count, count, 0, 0

    def arrive(self, n=1, expect_tx=0):
        self.tx += expect_tx
        self.pending -= n
        assert self.pending >= 0, "more arrivals than the barrier's count"
        self._settle()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._settle()

    def _settle(self):
        if self.pending == 0 and self.tx == 0:
            self.done += 1
            self.pending = self.count

    def passes(self, parity):
        # mbarrier.try_wait.parity: the phase of this parity has completed
        return (self.done & 1) != parity


class Ring:
    """StageRing's {stage, phase} cursor, plus the lap it stands for (the model's own bookkeeping)."""

    def __init__(self):
        self.stage = self.phase = self.lap = 0

    def advance(self):
        self.stage += 1
        if self.stage == STAGES:
            self.stage, self.phase, self.lap = 0, self.phase ^ 1, self.lap + 1

    def skip(self, n):
        self.stage += n
        laps = self.stage // STAGES
        self.stage -= laps * STAGES
        self.phase ^= laps & 1
        self.lap += laps


class Violation(AssertionError):
    pass


def check(cond, msg):
    if not cond:
        raise Violation(msg)


class Cta:
    def __init__(self, cluster, remote_release):
        n = 4 * (cluster if remote_release else 1)
        self.full = [Bar(1) for _ in range(STAGES)]
        self.empty = [Bar(n) for _ in range(STAGES)]
        self.order = [Bar(1), Bar(1)]    # four lane-0 arrivals of one warpgroup: one arrival here
        self.released = [0] * STAGES     # releases of each stage by this CTA's consumers
        self.multicasts = [0] * STAGES
        self.exited = False
        self.agents_left = 3


def wait(bar, parity, lo, hi, what):
    """A parity wait meant to pass once the barrier has completed `hi` phases.  While it polls, the barrier must be at
    `lo` = hi - 1 phases or more (at most one phase ahead of the waiter) and never past `hi`."""
    def poll():
        check(lo <= bar.done <= hi, f"{what}: barrier at phase {bar.done}, wait intends {hi} (parity aliasing)")
        ok = bar.passes(parity)
        check(ok == (bar.done >= hi), f"{what}: parity and intent disagree at phase {bar.done}")
        return ok
    return poll


def simulate(rows, B, N, segs, max_clusters, cluster=2, seed=0, w_kn=None, remote_release=True, final_sync=True,
             bm=128, bn=128):
    rng = random.Random(seed)
    tiles_per_batch = -(-rows // bm)
    tiles_m = tiles_per_batch * B
    tiles_n = -(-N // bn)
    units_m = -(-tiles_m // cluster)
    num_units = units_m * tiles_n
    nclusters = min(num_units, max_clusters)
    kblocks = [-(-k // 64) for k in segs]
    nk = sum(kblocks)
    w_kn = w_kn or [False] * len(segs)
    ctas = [[Cta(cluster, remote_release) for _ in range(cluster)] for _ in range(nclusters)]
    inflight = []      # (cluster id, rank, stage, lap, bytes)
    computed = []      # (tm, tn) per consumer tile
    sync_count = [0] * nclusters

    def tile_of(unit, rank):
        pm, tn = tile_coords(unit, units_m, tiles_n)
        return pm * cluster + rank, tn

    def producer(cid, rank):
        me = ctas[cid][rank]
        ring = Ring()
        for unit in range(cid, num_units, nclusters):
            for seg in range(len(segs)):
                for _ in range(kblocks[seg]):
                    s, lap = ring.stage, ring.lap
                    yield wait(me.empty[s], ring.phase ^ 1, lap - 1, lap, f"cluster {cid} rank {rank} empty[{s}]")
                    me.full[s].arrive(1, expect_tx=A_BYTES + W_BYTES)
                    inflight.append((cid, rank, s, lap, A_BYTES))
                    if cluster == 2:
                        me.multicasts[s] += 1
                        for dst in range(cluster):
                            inflight.append((cid, dst, s, lap, W_BYTES // 2))
                    else:
                        boxes = 2 if w_kn[seg] else 1
                        for _ in range(boxes):
                            inflight.append((cid, rank, s, lap, W_BYTES // boxes))
                    for dst in (range(cluster) if cluster == 2 else (rank,)):
                        t = ctas[cid][dst]
                        check(not t.exited, "TMA into an exited CTA")
                        check(t.released[s] >= lap, f"cluster {cid}: stage {s} of rank {dst} refilled (lap {lap}) "
                                                    "before its consumers released it")
                    ring.advance()

    def consumer(cid, rank, cw):
        me = ctas[cid][rank]
        peer = ctas[cid][rank ^ 1] if cluster == 2 else None
        ring = Ring()
        if cw == 1:
            ring.skip(nk)
        order_waits = 0
        for unit in range(cid + cw * nclusters, num_units, 2 * nclusters):
            if unit != cid:
                bar = me.order[cw]
                yield wait(bar, order_waits & 1, order_waits, order_waits + 1, f"order[{cw}]")
                order_waits += 1
            computed.append(tile_of(unit, rank))
            prev = -1
            for seg in range(len(segs)):
                for _ in range(kblocks[seg]):
                    s, lap = ring.stage, ring.lap
                    yield wait(me.full[s], ring.phase, lap, lap + 1, f"cluster {cid} rank {rank} full[{s}]")
                    if prev >= 0:
                        release(me, peer, prev)
                    prev = s
                    ring.advance()
            if unit + nclusters < num_units:
                me.order[cw ^ 1].arrive(1)
            ring.skip(nk)
            release(me, peer, prev)

    def release(me, peer, s):
        me.released[s] += 1
        me.empty[s].arrive(4)
        if peer is not None and remote_release:
            check(not peer.exited, "remote arrive on an exited CTA")
            peer.empty[s].arrive(4)

    def finish(cid, rank, gen):
        yield from gen
        if cluster == 2 and final_sync:
            sync_count[cid] += 1
            yield lambda: sync_count[cid] == 3 * cluster
        me = ctas[cid][rank]
        me.agents_left -= 1
        if me.agents_left == 0:
            check(not any(f[0] == cid and f[1] == rank for f in inflight), "CTA exits with a TMA copy still landing")
            me.exited = True

    agents = []
    for cid in range(nclusters):
        for rank in range(cluster):
            agents.append(finish(cid, rank, producer(cid, rank)))
            for cw in range(2):
                agents.append(finish(cid, rank, consumer(cid, rank, cw)))
    # a bias per CTA lets one CTA of a cluster run far ahead of its peer in some interleavings
    bias = [rng.choice((1, 1, 4, 30)) for _ in range(len(agents))]
    waiting = {}
    for i, a in enumerate(agents):
        waiting[i] = next(a, None)
    live = {i for i, w in waiting.items() if w is not None}
    while live or inflight:
        ready = [i for i in live if waiting[i]()]
        choices = [("a", i) for i in ready for _ in range(bias[i])] + [("t", j) for j in range(len(inflight))]
        if not choices:
            raise Violation(f"deadlock: {len(live)} agents wait and no copy is in flight")
        kind, i = rng.choice(choices)
        if kind == "t":
            cid, rank, s, lap, nbytes = inflight.pop(i)
            t = ctas[cid][rank]
            check(not t.exited, "TMA landed in an exited CTA")
            check(t.full[s].done == lap, f"bytes of lap {lap} landed on full[{s}] at phase {t.full[s].done}")
            t.full[s].complete_tx(nbytes)
            continue
        waiting[i] = next(agents[i], None)
        if waiting[i] is None:
            live.discard(i)

    for cid in range(nclusters):
        mc = [ctas[cid][r].multicasts for r in range(cluster)]
        check(all(m == mc[0] for m in mc), f"cluster {cid}: multicasts per stage differ {mc}")
    real = sorted(t for t in computed if t[0] < tiles_m)
    check(real == sorted((m, n) for m in range(tiles_m) for n in range(tiles_n)), "tiles not computed exactly once")
    phantom = [t for t in computed if t[0] >= tiles_m]
    check(all(t[0] == tiles_m for t in phantom), f"phantom tiles past the pair: {phantom}")
    check(len(phantom) == (tiles_n if cluster == 2 and tiles_m % 2 else 0), "phantom tile count")
    return {"units": num_units, "clusters": nclusters, "phantoms": len(phantom)}


SEEDS = range(12)
SEG7 = [200, 72, 16]       # 4 + 2 + 1 = 7 k-blocks: the ring is out of step at every tile boundary

CASES = {
    # name: (rows per batch, batches, N, segments, clusters on the device)
    "tiles_m1": (128, 1, 512, SEG7, 4),
    "tiles_m2": (256, 1, 512, SEG7, 4),
    "tiles_m3": (300, 1, 512, SEG7, 4),
    "even_tiles_m_b3": (200, 3, 384, SEG7, 4),    # 2 m-tiles per batch: pairs align with the batches
    "odd_tiles_m_b3": (300, 3, 384, SEG7, 4),     # 3 per batch, 9 in all: pairs straddle batch boundaries, one phantom
    "odd_tiles_m_b5": (100, 5, 256, SEG7, 3),     # 1 per batch: every pair straddles
    "fewer_pairs_than_clusters": (256, 1, 384, SEG7, 4),
    "one_pair_per_cluster": (256, 1, 512, SEG7, 4),
    "one_extra_pair": (256, 1, 640, SEG7, 4),
    "three_pairs_per_cluster": (768, 1, 512, SEG7, 4),
    "one_segment": (512, 1, 512, [448], 3),
    "two_segments": (384, 2, 512, [3072, 16], 5),
    "deep_k": (512, 1, 256, [12288 // 16], 2),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("w_kn", (False, True))
def test_cluster_protocol(case, w_kn):
    rows, B, N, segs, clusters = CASES[case]
    for seed in SEEDS:
        simulate(rows, B, N, segs, clusters, seed=seed, w_kn=[w_kn] * len(segs))


def test_case_shapes_cover_the_pair_counts():
    got = {k: simulate(r, b, n, s, c) for k, (r, b, n, s, c) in CASES.items()}
    assert all(got[k]["phantoms"] > 0 for k in ("tiles_m1", "tiles_m3", "odd_tiles_m_b3", "odd_tiles_m_b5"))
    assert got["even_tiles_m_b3"]["phantoms"] == 0
    assert got["fewer_pairs_than_clusters"]["units"] < 4
    assert got["one_pair_per_cluster"]["units"] == 4
    assert got["one_extra_pair"]["units"] == 5
    assert got["three_pairs_per_cluster"]["units"] == 12 and got["three_pairs_per_cluster"]["clusters"] == 4


@pytest.mark.parametrize("case", ("tiles_m2", "odd_tiles_m_b3", "one_extra_pair"))
def test_single_cta_kernel_rules(case):
    rows, B, N, segs, clusters = CASES[case]
    for seed in SEEDS:
        simulate(rows, B, N, segs, clusters, cluster=1, seed=seed)


def _finds_violation(**kw):
    rows, B, N, segs, clusters = CASES["three_pairs_per_cluster"]
    for seed in range(200):
        try:
            simulate(rows, B, N, segs, clusters, seed=seed, **kw)
        except Violation:
            return True
    return False


def test_model_catches_a_producer_that_waits_for_its_own_consumers_only():
    assert _finds_violation(remote_release=False)


def test_model_catches_an_exit_without_the_cluster_sync():
    assert _finds_violation(final_sync=False)
