"""Protocol model of the K4 stage hand-off (csrc/maxpool_tc.cu): producers -> ring of MP_SA stages -> MMA warp, with the
same slot / parity arithmetic as the kernels, driven by a random scheduler.  It checks the things a hang or a silent
corruption on the GPU would come from: no deadlock, no wait satisfied by an aliased (two phases old) parity, no stage
refilled before its MMAs retired, every K-block consumed exactly once and in order - for the default kernel's
row-split producers, the gather4 variant's stage-per-warp producers and the cluster-multicast variant.

An mbarrier is modelled with what the hardware keeps: a pending-arrival count, a transaction count and ONE phase bit;
`wait(parity)` succeeds when the current phase bit differs from `parity` (the phase with that parity has completed).
The model additionally tracks the true number of completed phases to flag aliasing.

    python tools/pipeline_model.py            # sweep of configurations, prints a summary
"""
import random


class MBarrier(object):
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase, self.completed = count, count, 0, 0, 0

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phase ^= 1
            self.completed += 1
            self.pending = self.count

    def arrive(self, expect_tx=0):
        assert self.pending > 0, "more arrivals than the barrier's count in one phase"
        self.tx += expect_tx
        self.pending -= 1
        self._maybe_complete()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._maybe_complete()

    def ready(self, parity, expected_completed):
        """hardware test + aliasing check: the caller states how many completed phases it is really waiting for"""
        ok = self.phase != parity
        if ok:
            assert self.completed == expected_completed, \
                "parity aliasing: wait passed with %d completed phases, wanted %d" % (self.completed, expected_completed)
        return ok


class Cta(object):
    def __init__(self, sa, cl):
        self.full = [MBarrier(1) for _ in range(sa)]        # own expect_tx arrive (+ transactions)
        self.empty = [MBarrier(cl) for _ in range(sa)]      # one (multicast) commit per CTA of the cluster
        self.content = [None] * sa                          # K-block index held by the stage
        self.retired = [True] * sa                          # the MMAs that read the stage have completed
        self.bytes_of = [0] * sa
        self.consumed = 0


def simulate(kind, sa, total_it, n_prod, cl=1, seed=0, stage_bytes=8192, max_steps=2000000):
    """kind: 'groups' (round-2 cp.async producers: n_prod warps in two groups; group g fills the stages it = g, g + 2, ...
    and each of its warps arrives once per stage), 'rowsplit' (default kernel: every producer warp fills its rows of EVERY stage, lagged publish not modelled:
    arrive per warp), 'g4' (warp w fills whole stages it = w, w + n_prod, ...; the kernels use n_prod == sa), 'g4mc' (as g4 in each of cl CTAs, each
    issuing 1/cl of every stage to all CTAs).  Returns the number of scheduler steps."""
    rnd = random.Random(seed)
    ctas = [Cta(sa, cl if kind == "g4mc" else 1) for _ in range(cl if kind == "g4mc" else 1)]
    if kind == "rowsplit":
        for c in ctas:
            c.full = [MBarrier(n_prod) for _ in range(sa)]
    if kind == "groups":
        for c in ctas:
            c.full = [MBarrier(n_prod // 2) for _ in range(sa)]
    inflight = []                                           # delayed events: (fire_step, fn)
    step = [0]

    def later(fn):
        inflight.append((step[0] + rnd.randint(1, 40), fn))

    # ---- agents as generators: yield a predicate to wait on, or None to just take a step
    def producer(ci, w):
        c = ctas[ci]
        if kind == "rowsplit":
            its = range(total_it)
        elif kind == "groups":
            its = range(w // (n_prod // 2), total_it, 2)         # the warp's group takes every other K-block
        else:
            its = range(w, total_it, n_prod)
        for it in its:
            s, n = it % sa, it // sa
            yield lambda: c.empty[s].ready((n & 1) ^ 1, n)
            if kind in ("rowsplit", "groups"):
                if w % (n_prod // 2 if kind == "groups" else n_prod) == 0:
                    assert c.retired[s], "stage refilled before its MMAs retired"
                    c.content[s], c.retired[s] = it, False
                later(lambda s=s: c.full[s].arrive())            # copies land, fence, arrive
            else:
                share = stage_bytes // len(ctas)
                c.full[s].arrive(expect_tx=stage_bytes)          # lane 0: arrive.expect_tx for the whole stage
                for dst in (ctas if kind == "g4mc" else [c]):
                    def land(dst=dst, s=s, it=it, share=share):
                        if dst.bytes_of[s] == 0:
                            assert dst.retired[s], "stage refilled before its MMAs retired"
                            dst.content[s], dst.retired[s] = it, False
                        assert dst.content[s] == it, "two different K-blocks written into one stage"
                        dst.bytes_of[s] += share
                        if dst.bytes_of[s] == stage_bytes:
                            dst.bytes_of[s] = 0
                        dst.full[s].complete_tx(share)
                    later(land)
            yield None

    def mma(ci):
        c = ctas[ci]
        for it in range(total_it):
            s, n = it % sa, it // sa
            yield lambda: c.full[s].ready(n & 1, n + 1)
            assert c.content[s] == it, "MMA read K-block %r, expected %d" % (c.content[s], it)
            c.consumed += 1

            def retire(s=s):
                c.retired[s] = True
                for dst in (ctas if kind == "g4mc" else [c]):
                    dst.empty[s].arrive()                        # the MMA commit (multicast in the cluster form)
            later(retire)
            yield None

    agents = []
    for ci in range(len(ctas)):
        agents += [producer(ci, w) for w in range(n_prod)] + [mma(ci)]
    waiting = [None] * len(agents)
    alive = [True] * len(agents)
    while any(alive) or inflight:
        step[0] += 1
        assert step[0] < max_steps, "no progress: deadlock (or livelock) in the hand-off"
        due = [e for e in inflight if e[0] <= step[0]]
        if due:
            e = rnd.choice(due)
            inflight.remove(e)
            e[1]()
        order = [i for i in range(len(agents)) if alive[i]]
        rnd.shuffle(order)
        progressed = False
        for i in order:
            if waiting[i] is not None and not waiting[i]():
                continue
            try:
                waiting[i] = next(agents[i])
            except StopIteration:
                alive[i] = False
            progressed = True
            break
        if not progressed and not inflight and any(alive):
            raise AssertionError("deadlock: every agent is waiting and nothing is in flight")
    for c in ctas:
        assert c.consumed == total_it
    return step[0]


def sweep(seeds=3):
    """Every (ring size, K-blocks per tile, tiles) shape the kernels see, incl. fewer K-blocks than slots."""
    n = 0
    for sa in (6, 7):
        for kblocks, tiles in ((19, 3), (20, 2), (2, 9), (1, 13), (7, 4)):
            total = kblocks * tiles
            for seed in range(seeds):
                simulate("rowsplit", sa, total, 4, seed=seed)
                simulate("g4", sa, total, sa, seed=seed)                  # one producer warp per slot
                for cl in (2, 4):
                    simulate("g4mc", sa, total, sa, cl=cl, seed=seed)
                n += 4
    return n


def sweep_round2(seeds=2):
    """The round-2 kernels: two-group cp.async producers over 4 / 8 / 12 / 14 stages (maxpool_mlp_tmem_kernel, wide), and the
    cluster kernel - 4 producer warps, warp w owns the slots w, w + 4, ... of a ring whose size is a multiple of 4, clusters
    of 2 and 4 CTAs, multicast fills and multicast commits (maxpool_mlp_tmemc_kernel)."""
    n = 0
    for kblocks, tiles in ((10, 3), (4, 5), (1, 9), (19, 2)):
        total = kblocks * tiles
        for seed in range(seeds):
            for sa in (4, 8, 12, 14):
                simulate("groups", sa, total, 8, seed=seed)
                n += 1
            for sa in (4, 8, 12):
                for cl in (2, 4):
                    simulate("g4mc", sa, total, 4, cl=cl, seed=seed, stage_bytes=16384)
                    n += 1
    return n


def cluster_ring_must_be_a_multiple_of_the_producer_warps():
    """4 stage-filling warps over a 6-slot ring: a slot changes owner from fill to fill, a wait can pass on a stale phase."""
    try:
        for seed in range(30):
            simulate("g4mc", 6, 10 * 4, 4, cl=2, seed=seed, stage_bytes=16384)
    except AssertionError as e:
        return str(e)
    return None


def shows_the_aliasing_bug():
    """The design this model rejected: 8 stage-filling warps over 7 slots - a warp can be two fills ahead of a slot."""
    try:
        for seed in range(20):
            simulate("g4", 7, 19 * 3, 8, seed=seed)
    except AssertionError as e:
        return str(e)
    return None


if __name__ == "__main__":
    print("hand-off protocol model: %d simulations, no deadlock / aliasing / early refill / misordered K-block" % sweep())
    print("8 warps over 7 slots ->", shows_the_aliasing_bug())
    print("round-2 kernels: %d simulations clean" % sweep_round2())
    print("4 warps over a 6-slot cluster ring ->", cluster_ring_must_be_a_multiple_of_the_producer_warps())


def check_producer_walk(sa, kblocks, tiles):
    """The gather4 producers' incremental (tile, K-block) walk and their current / next-tile row-id registers
    (maxpool_mlp_g4_kernel: kb += MP_SA; while (kb >= kblocks) ...; adv == 1 -> cur = nxt) against the direct
    it // kblocks, it % kblocks.  `load` records which tile's ids a register set holds."""
    total = kblocks * tiles
    for warp in range(sa):
        tl, kb = 0, warp
        while kb >= kblocks:
            kb -= kblocks
            tl += 1
        cur, nxt = tl, tl + 1                       # load_ids(tl, cur); load_ids(tl + 1, nxt)
        it = warp
        while it < total:
            assert (cur, kb) == (it // kblocks, it % kblocks), (sa, kblocks, warp, it, cur, kb)
            kb += sa
            adv = 0
            while kb >= kblocks:
                kb -= kblocks
                adv += 1
            if adv == 1:
                cur = nxt
                tl += 1
                nxt = tl + 1
            elif adv > 1:
                tl += adv
                cur, nxt = tl, tl + 1
            it += sa
    return True
