"""Discrete models of mbarrier protocols (roles as coroutines, random interleavings): the channel-major forward kernel
explored for an earlier tensor-core design (tools/experiments/cca_tc_fwdt.cu, not adopted), and the backward kernel's load
ring, bulk copies and per-sample counters (ccnet_b200/csrc/cca_tc_bwd.cuh; build_bwd / run_bwd).

Not a performance model: it only answers "can this hand-shake deadlock, and does every arrive / wait hit the barrier
phase it was meant for?" before GPU minutes are spent on it.  Every wait and arrive carries the use index the code
derives its parity from; the model checks the parity formula against the barrier's real phase count.

  python tools/pipeline_model.py [NCH] [kNLd] [items] [seeds]
"""
import random
import sys


PROGRESS = [0]


class Bar:
    def __init__(self, name, count):
        self.name, self.count, self.done, self.pending = name, count, 0, 0

    def arrive(self, n=1, use=None):
        if use is not None and use != self.done:
            raise AssertionError(f"{self.name}: arrive for use {use} while phase {self.done} is open")
        PROGRESS[0] += 1
        self.pending += n
        if self.pending > self.count:
            raise AssertionError(f"{self.name}: over-arrival")
        if self.pending == self.count:
            self.pending = 0
            self.done += 1

    def ready(self, parity):                     # mbarrier.try_wait.parity
        return (self.done & 1) != parity


class NamedBar:                                  # bar.sync id, n  (n agents of equal weight)
    def __init__(self, n):
        self.n, self.gen, self.cnt = n, 0, 0


def wait(bar, parity, use=None):
    """use = number of completed phases the caller expects to need (parity must equal (use-1)&1 ... checked below)"""
    while not bar.ready(parity):
        yield
    if use is not None and bar.done != use:
        raise AssertionError(f"{bar.name}: wait expected {use} completed phases, barrier has {bar.done}")


def sync(nb):
    g = nb.gen
    nb.cnt += 1
    if nb.cnt == nb.n:
        nb.cnt = 0
        nb.gen += 1
    while nb.gen == g:
        yield


def build(NCH, kNLd, nk):
    NG = NCH // 2
    qkpos = 2 if NCH >= 3 else NCH - 1
    B = {}
    for i in range(kNLd):
        B["LD_FULL", i] = Bar(f"LD_FULL{i}", 1)
        B["LD_EMPTY", i] = Bar(f"LD_EMPTY{i}", 1)
        B["OP_FULL", i] = Bar(f"OP_FULL{i}", 512)
    B["S_FULL"] = Bar("S_FULL", 1)
    B["S_EMPTY"] = Bar("S_EMPTY", 128)
    for i in range(2):
        B["P_FULL", i] = Bar(f"P_FULL{i}", 128)
        B["P_EMPTY", i] = Bar(f"P_EMPTY{i}", 1)
        B["V_FULL", i] = Bar(f"V_FULL{i}", 512)
        B["V_EMPTY", i] = Bar(f"V_EMPTY{i}", 1)
        B["O_FULL", i] = Bar(f"O_FULL{i}", 1)
        B["O_EMPTY", i] = Bar(f"O_EMPTY{i}", 128)
    rd_cnt = [0] * kNLd
    nb = {1: NamedBar(2), 3: NamedBar(2)}        # two model agents (half 0 / half 1 warps) per 256-thread group
    # ring: list of (kind, item, chunk)
    ring = [("Q", 0, 0), ("K", 0, 0)]
    for k in range(nk):
        for n in range(NCH):
            if n == qkpos and k + 1 < nk:
                ring += [("Q", k + 1, 0), ("K", k + 1, 0)]
            ring.append(("V", k, n))
    uses = {}                                    # ring index -> completed phases LD_FULL/LD_EMPTY expect

    def producer():
        for g, _ in enumerate(ring):
            slot = g % kNLd
            yield from wait(B["LD_EMPTY", slot], ((g // kNLd) & 1) ^ 1, g // kNLd)
            B["LD_FULL", slot].arrive(use=g // kNLd)

    def mma():
        u = gc = 0
        qkpar = 0
        opuse = [0] * kNLd

        def issue_s(k):
            nonlocal u, qkpar
            sq, sk = u % kNLd, (u + 1) % kNLd
            assert ring[u][0] == "Q" and ring[u + 1][0] == "K" and ring[u][1] == k, (u, ring[u], k)
            for s in (sq, sk):
                yield from wait(B["OP_FULL", s], (qkpar >> s) & 1, opuse[s] + 1)
                opuse[s] += 1
            qkpar ^= (1 << sq) | (1 << sk)
            yield from wait(B["S_EMPTY"], (k & 1) ^ 1, k)
            B["S_FULL"].arrive(use=k)
            B["LD_EMPTY", sq].arrive(use=u // kNLd)
            B["LD_EMPTY", sk].arrive(use=(u + 1) // kNLd)
            u += 2

        if nk > 0:
            yield from issue_s(0)
        for k in range(nk):
            yield from wait(B["P_FULL", k & 1], (k >> 1) & 1, (k >> 1) + 1)
            for g in range(NG):
                for h in range(2):
                    if 2 * g + h == qkpos and k + 1 < nk:
                        yield from issue_s(k + 1)
                    assert ring[u] == ("V", k, 2 * g + h), (u, ring[u], k, g, h)
                    u += 1
                vb = gc & 1
                yield from wait(B["V_FULL", vb], (gc >> 1) & 1, (gc >> 1) + 1)
                for hb in range(2):
                    yield from wait(B["O_EMPTY", hb], (gc & 1) ^ 1, gc)
                    yield                                   # (commit arrives some time later)
                    B["O_FULL", hb].arrive(use=gc)
                yield
                B["V_EMPTY", vb].arrive(use=gc >> 1)
                gc += 1
            B["P_EMPTY", k & 1].arrive(use=k >> 1)

    def converter(grp, half):                    # 128 threads = 4 warps: weight 128 on the 512-count barriers
        g = 0
        pend = [-1]

        def publish():
            if pend[0] >= 0:
                B["OP_FULL", pend[0]].arrive(128)
                pend[0] = -1

        def wait_full(slot, gg):
            if not B["LD_FULL", slot].ready((gg // kNLd) & 1):
                publish()
            yield from wait(B["LD_FULL", slot], (gg // kNLd) & 1, gg // kNLd + 1)

        def conv_qk(count):
            nonlocal g
            for _ in range(count):
                slot = g % kNLd
                assert ring[g][0] in "QK"
                yield from wait_full(slot, g)
                publish()                                    # mid()
                yield from sync(nb[1 if grp == 0 else 3])
                pend[0] = slot
                g += 1

        def conv_v(n, gcn):
            nonlocal g
            slot = g % kNLd
            assert ring[g][0] == "V" and ring[g][2] == n
            if (n & 1) == half:
                yield from wait_full(slot, g)
                publish()
                yield
                rd_cnt[slot] += 4                            # the slot goes back before the wait for the TMEM buffer
                if rd_cnt[slot] == 8:
                    rd_cnt[slot] = 0
                    B["LD_EMPTY", slot].arrive(use=g // kNLd)
                vb = gcn & 1
                yield from wait(B["V_EMPTY", vb], ((gcn >> 1) & 1) ^ 1, gcn >> 1)
                yield
                B["V_FULL", vb].arrive(128, use=gcn >> 1)
            g += 1

        if nk > 0:
            yield from conv_qk(2)
        gcn = 0
        for k in range(nk):
            for n in range(NCH):
                if n == qkpos and k + 1 < nk:
                    yield from conv_qk(2)
                yield from conv_v(n, gcn + (n >> 1))
                if n == NCH - 1:
                    gcn += NG
        publish()

    def softmax():
        for k in range(nk):
            yield from wait(B["S_FULL"], k & 1, k + 1)
            yield from wait(B["P_EMPTY", k & 1], ((k >> 1) & 1) ^ 1, k >> 1)
            yield
            B["P_FULL", k & 1].arrive(128, use=k >> 1)
            B["S_EMPTY"].arrive(128, use=k)

    def epilogue():
        gc = 0
        for k in range(nk):
            for g in range(NG):
                for hb in range(2):
                    yield from wait(B["O_FULL", hb], gc & 1, gc + 1)
                    yield
                    B["O_EMPTY", hb].arrive(128, use=gc)
                gc += 1

    agents = {"producer": producer(), "mma": mma(), "softmax": softmax(), "epilogue": epilogue()}
    for grp in range(2):
        for half in range(2):
            agents[f"conv{grp}{half}"] = converter(grp, half)
    return agents


def run(NCH, kNLd, nk, seed):
    rng = random.Random(seed)
    agents = build(NCH, kNLd, nk)
    live = dict(agents)
    idle, last = 0, PROGRESS[0]
    names = list(live)
    weights = {n: rng.choice((1, 1, 1, 5, 25)) for n in names}      # biased schedules: some roles much faster than others
    while live:
        name = rng.choices(names, [weights[n] for n in names])[0]
        try:
            next(live[name])
        except StopIteration:
            del live[name]
            names.remove(name)
        if PROGRESS[0] != last:
            last, idle = PROGRESS[0], 0
        else:
            idle += 1
        if idle > 20000:
            raise AssertionError(f"deadlock: still running {sorted(live)}")
    return True


# ---------------------------------------------------------------------------------------------------------------------------
# Backward kernel (ccnet_b200/csrc/cca_tc_bwd.cuh): the load ring, the bulk copies and the per-sample counters, over several CTAs.
#
# Per CTA two roles: the producer lane (it waits only on ring slots) and the consumers (the 256 threads move together through
# their barriers, so one agent; thread 0's arrivals are its events).  A third agent per CTA plays the bulk-copy engine: it
# reads the committed groups in order and completes their writes some time later.  Items are those of cca_items.cuh with one
# tile per line (column items store and publish, row items add after the counter), in the real item orders.

def bwd_items(B, H, W, lag):
    """[(b, producer)] in the order of decode_item / decode_item_lagged (one tile per line: seg1 is empty)."""
    seg0, per_sample = W, W + H
    def in_sample(b, j):
        return (b, j < seg0)
    out = []
    for idx in range(B * per_sample):
        if not lag:
            out.append(in_sample(idx // per_sample, idx % per_sample))
            continue
        if idx < seg0:
            out.append(in_sample(0, idx))
            continue
        x = idx - seg0
        grp, rem = divmod(x, per_sample)
        if grp < B - 1:
            out.append(in_sample(grp + 1, rem) if rem < seg0 else in_sample(grp, rem))
        else:
            out.append(in_sample(B - 1, seg0 + rem))
    return out, seg0


def build_bwd(kNLd, NCH, B, H, W, ncta, lag, nqk=4, publish="before_waits"):
    """nqk: ring entries of an item's Q and K (4 in fp32, 2 for 16-bit I/O).  publish: where a producer item's count is
    published -- "before_waits" (the kernel: in the next item, after S, before its first counter wait) or "after_wait" (after
    the next item's first counter wait: must deadlock when a CTA consumes the sample it just produced)."""
    items, seg0 = bwd_items(B, H, W, lag)
    cdone, ddone = [0] * B, [0] * B
    agents = {}

    def count_wait(cnt, b):
        while cnt[b] < seg0:
            yield

    def bump(cnt, b):
        PROGRESS[0] += 1
        cnt[b] += 1

    for c in range(ncta):
        mine = items[c::ncta]
        full = [Bar(f"c{c}.full{i}", 1) for i in range(kNLd)]
        empty = [Bar(f"c{c}.empty{i}", 1) for i in range(kNLd)]
        bulk = {"groups": [], "read": 0, "written": 0}     # committed groups (kind), how many read / written so far
        region = {"dq_group": -1}                           # the group of the last dQ copy out of the K region

        def producer(mine=mine, full=full, empty=empty):
            g = 0
            for b, prod in mine:
                for _ in range(nqk + (3 if prod else 2) * NCH):   # Q, K boxes; per chunk V, dO (, O: delta producers)
                    slot = g % kNLd
                    yield from wait(empty[slot], ((g // kNLd) & 1) ^ 1, g // kNLd)
                    yield                                          # (the TMA lands some time later)
                    full[slot].arrive(use=g // kNLd)
                    g += 1

        def engine(bulk=bulk, rng=random.Random(c)):
            while not bulk.get("done"):                      # reads in commit order; a group's writes complete after its read
                yield
                can_read, can_write = bulk["read"] < len(bulk["groups"]), bulk["written"] < bulk["read"]
                if can_read and (not can_write or rng.random() < 0.5):
                    bulk["read"] += 1
                    PROGRESS[0] += 1
                elif can_write:
                    bulk["written"] += 1
                    PROGRESS[0] += 1

        def consumer(mine=mine, full=full, empty=empty, bulk=bulk, region=region):
            g = 0
            pending = -1
            unpublished = -1

            def commit(kind):
                bulk["groups"].append(kind)
                return len(bulk["groups"]) - 1

            def wait_read(n):                                    # cp.async.bulk.wait_group.read n
                while len(bulk["groups"]) - bulk["read"] > n:
                    yield

            def wait_written():                                  # cp.async.bulk.wait_group 0
                while bulk["written"] < len(bulk["groups"]):
                    yield

            def wfull(gi):
                yield from wait(full[gi % kNLd], (gi // kNLd) & 1, gi // kNLd + 1)

            def publish_if_due():
                nonlocal unpublished
                if unpublished >= 0:
                    yield from wait_written()
                    bump(cdone, unpublished)
                    unpublished = -1

            for b, prod in mine:
                calc = prod                                      # delta mode 1: the column items of the first key block
                per = 3 if calc else 2
                # Q, K entries -> the Q / K region (after the barrier that follows the previous item's dQ wait_group.read)
                for i in range(nqk):
                    yield from wfull(g + i)
                if region["dq_group"] >= 0 and bulk["read"] <= region["dq_group"]:
                    raise AssertionError("Q / K region written while the previous dQ copy may still read it")
                yield
                for i in range(nqk):
                    empty[(g + i) % kNLd].arrive(use=(g + i) // kNLd)
                g += nqk
                # S; then the deferred publish (or the wait for the dK copy's read of the P planes)
                yield
                if publish == "before_waits":
                    yield from publish_if_due()
                yield from wait_read(0)

                def convert(n):
                    gv = g + per * n
                    yield from wfull(gv)
                    yield from wfull(gv + 1)
                    if calc:
                        yield from wfull(gv + 2)
                        yield
                        empty[(gv + 2) % kNLd].arrive(use=(gv + 2) // kNLd)

                yield from convert(0)
                for n in range(NCH):
                    if n + 1 < NCH:
                        yield from convert(n + 1)
                    if pending >= 0:                             # release(): the previous dV copy has read its dO slot
                        yield from wait_read(0)
                        empty[pending % kNLd].arrive(use=pending // kNLd)
                        pending = -1
                    yield                                        # wg_wait<0>
                    if n == 0 and not prod:
                        yield from count_wait(cdone, b)
                        if publish == "after_wait":
                            yield from publish_if_due()
                    gv = g + per * n
                    empty[gv % kNLd].arrive(use=gv // kNLd)      # V free
                    yield                                        # dP(n + 1) issued, dV(n) staged in the dO slot
                    commit("dv")
                    pending = gv + 1
                g += per * NCH
                if calc:
                    bump(ddone, b)
                else:
                    yield from count_wait(ddone, b)
                    if publish == "after_wait":
                        yield from publish_if_due()
                yield                                            # dS, dQ MMAs
                region["dq_group"] = commit("dq")
                yield                                            # dK MMAs
                commit("dk")
                yield from wait_read(1)
                if pending >= 0:
                    empty[pending % kNLd].arrive(use=pending // kNLd)
                    pending = -1
                if prod:
                    unpublished = b
            yield from wait_written()
            yield from publish_if_due()
            bulk["done"] = True

        agents[f"prod{c}"] = producer()
        agents[f"cons{c}"] = consumer()
        agents[f"bulk{c}"] = engine()
    return agents, cdone, ddone, seg0


def run_bwd(kNLd, NCH, B, H, W, ncta, lag, seed, nqk=4, publish="before_waits"):
    rng = random.Random(seed)
    agents, cdone, ddone, seg0 = build_bwd(kNLd, NCH, B, H, W, ncta, lag, nqk, publish)
    live = dict(agents)
    names = list(live)
    weights = {n: rng.choice((1, 1, 1, 5, 25)) for n in names}
    idle, last = 0, PROGRESS[0]
    while live:
        name = rng.choices(names, [weights[n] for n in names])[0]
        try:
            next(live[name])
        except StopIteration:
            del live[name]
            names.remove(name)
        if PROGRESS[0] != last:
            last, idle = PROGRESS[0], 0
        else:
            idle += 1
        if idle > 20000:
            raise AssertionError(f"deadlock: still running {sorted(live)}")
    if cdone != [seg0] * B or ddone != [seg0] * B:
        raise AssertionError(f"counters {cdone} {ddone}, expected {seg0} each")
    return True


if __name__ == "__main__":
    NCH = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    kNLd = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    nk = int(sys.argv[3]) if len(sys.argv) > 3 else 6
    seeds = int(sys.argv[4]) if len(sys.argv) > 4 else 200
    for s in range(seeds):
        run(NCH, kNLd, nk, s)
    print(f"ok: NCH={NCH} slots={kNLd} items={nk} seeds={seeds}")
