"""Executable model of the attention kernels' warp / mbarrier protocols (CPU, no GPU).

Why: round 1 shipped a dQ kernel whose lane quarters were coupled through ONE "dS ready" mbarrier
shared by two TMEM stages; a quarter running a block ahead completed the phase for a slower one and
the dQ MMA consumed stale data in 1.2 % of launches (DESIGN.md 6). Every parity test passed. The
protocol, not the arithmetic, was wrong -- and a protocol can be checked on a CPU by running it
under adversarial schedules with tagged buffer contents.

Model: agents are generators that yield blocking conditions; a random scheduler picks any runnable
agent, with arbitrary stalls. `Mbar` follows PTX mbarrier semantics (pending-arrival count, phase
bit, try_wait on parity). The tensor pipe is an in-order queue of issued ops (MMAs and commits)
that an extra agent retires one at a time, so `tcgen05.commit` arrives only after everything issued
before it has executed. Buffers carry tags ("what is in here"); every consumer asserts the tag it
needs. A run ends in OK, a Violation (stale / overwritten data) or a deadlock.

The first models below are the protocols of the earlier tcgen05 kernels (an MMA warp, tensor memory, staging
tiles): the v9 / v10 dQ kernel, the dK/dV and forward kernels and the CTA-pair GEMM. They stay as the record of
what the model found and as checks of its sensitivity. The sm_90a kernels that ship now (wgmma, a TMA
producer and consumer warpgroups) share one operand-ring protocol, modelled by `wg_ring_kernel`. tests/test_protocol_model.py requires
that the model FINDS the v9 bug. It also found something nobody had seen on hardware: the shipped
dK/dV protocol (one bar_p) is free of stale reads but not of an ABA deadlock -- if the MMA warp is
held up for a whole compute iteration right after issuing the next block's score MMAs, the compute
warps finish two blocks, bar_p flips twice and the MMA warp waits for a phase that is already gone.
Real warps do not stall like the model's scheduler, so this needs an external stall to happen
(DESIGN.md 7 discusses whether the 8-GPU failure was one); bar_p per stage removes it."""
import random


class Violation(Exception):
    pass


class Mbar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):          # mbarrier.try_wait.parity: true once the phase `parity` completed
        return self.phase != parity


class TensorPipe:
    """in-order execution of issued tcgen05 ops"""

    def __init__(self):
        self.q = []

    def issue(self, fn):
        self.q.append(fn)

    def commit(self, bar):
        self.q.append(bar.arrive)

    def agent(self, done):
        while True:
            if self.q:
                self.q.pop(0)()
                yield None
            elif done():
                return
            else:
                yield (lambda: bool(self.q) or done())


def run(agents, rng, max_steps=200000, stall_p=0.15):
    """agents: dict name -> generator. Generators yield None (runnable again) or a predicate to
    wait on. Random scheduling with random multi-step stalls."""
    waiting = {n: None for n in agents}
    stalled = {n: 0 for n in agents}
    live = dict(agents)
    for _ in range(max_steps):
        if not live:
            return "ok"
        runnable = [n for n in live if stalled[n] == 0 and (waiting[n] is None or waiting[n]())]
        any_stalled = any(stalled[n] for n in live)
        for n in live:
            if stalled[n]:
                stalled[n] -= 1
        if not runnable:
            if not any_stalled:      # nobody can move and nobody is merely descheduled
                return "deadlock: " + ", ".join(sorted(live))
            continue
        n = rng.choice(runnable)
        if rng.random() < stall_p:                      # this agent loses its SM sub-partition for a while
            stalled[n] = rng.randint(1, 40)
        try:
            waiting[n] = next(live[n])
        except StopIteration:
            del live[n]
    return "step limit"


# ---------------------------------------------------------------------------------------------
# dQ kernel (attention.cu attn_bwd_dq_kernel): MMA warp + 4 lane quarters (x hc collapsed) + tensor pipe
# ---------------------------------------------------------------------------------------------
def dq_kernel(njb, per_stage_bar_p, rng, quarters=4, threads_per_quarter=2):
    n_thr = quarters * threads_per_quarter
    pipe = TensorPipe()
    bar_s = [Mbar(1), Mbar(1)]
    bar_p = [Mbar(n_thr), Mbar(n_thr)] if per_stage_bar_p else [Mbar(n_thr)]
    bar_dq = Mbar(1)
    # tags: S[tb] = block whose scores are there; dS[tb][q][t] = block whose dS that thread wrote
    S = [None, None]
    dS = [[[None] * threads_per_quarter for _ in range(quarters)] for _ in range(2)]
    state = dict(mma_done=False, dq_blocks=[])

    def scores(j):
        def ex():
            S[j & 1] = j
            for q in range(quarters):                  # the dP MMA overwrites the columns dS lives in
                for t in range(threads_per_quarter):
                    dS[j & 1][q][t] = ("dP", j)
        return ex

    def dq_mma(j):
        def ex():
            for q in range(quarters):
                for t in range(threads_per_quarter):
                    if dS[j & 1][q][t] != ("dS", j):
                        raise Violation(f"dQ MMA of block {j} read {dS[j & 1][q][t]} from quarter {q}")
            state["dq_blocks"].append(j)
        return ex

    def mma_warp():
        pipe.issue(scores(0)); pipe.commit(bar_s[0])
        yield None
        for j in range(njb):
            if j + 1 < njb:
                pipe.issue(scores(j + 1)); pipe.commit(bar_s[(j + 1) & 1])
                yield None
            if per_stage_bar_p:
                b, par = bar_p[j & 1], (j >> 1) & 1
            else:
                b, par = bar_p[0], j & 1
            yield (lambda b=b, par=par: b.passed(par))
            pipe.issue(dq_mma(j))
            if j + 1 == njb:
                pipe.commit(bar_dq)
            yield None
        state["mma_done"] = True

    def compute(q, t):
        for j in range(njb):
            tb = j & 1
            yield (lambda tb=tb, j=j: bar_s[tb].passed((j >> 1) & 1))
            if S[tb] != j:
                raise Violation(f"quarter {q} read scores of block {S[tb]} while working on block {j}")
            yield None                                  # exp / dS math
            dS[tb][q][t] = ("dS", j)                    # tcgen05.st over the dP columns
            yield None
            (bar_p[tb] if per_stage_bar_p else bar_p[0]).arrive()
            yield None
        yield (lambda: bar_dq.passed(0))

    agents = {"mma": mma_warp(), "pipe": pipe.agent(lambda: state["mma_done"])}
    for q in range(quarters):
        for t in range(threads_per_quarter):
            agents[f"q{q}t{t}"] = compute(q, t)
    res = run(agents, rng)
    if res == "ok" and state["dq_blocks"] != list(range(njb)):
        raise Violation(f"dQ blocks executed: {state['dq_blocks']}")
    return res


# ---------------------------------------------------------------------------------------------
# dK/dV kernel (attn_bwd_dkdv_kernel): TMA warp (3 Q/dO buffers), MMA warp, compute warps with a
# block-wide barrier every iteration, staging tiles double-buffered behind bar_d
# ---------------------------------------------------------------------------------------------
def dkdv_kernel(n_iter, rng, n_thr=6, block_barrier=True, per_stage_bar_p=False):
    pipe = TensorPipe()
    bar_q = [Mbar(1) for _ in range(3)]
    bar_qfree = [Mbar(1) for _ in range(3)]
    bar_s, bar_d = [Mbar(1), Mbar(1)], [Mbar(1), Mbar(1)]
    bar_p = [Mbar(n_thr), Mbar(n_thr)] if per_stage_bar_p else [Mbar(n_thr)]
    Q = [None] * 3                       # which block's Q/dO is in buffer b
    S = [None, None]
    stage = [[None] * n_thr for _ in range(2)]     # P/dS staging tiles
    state = dict(mma_done=False, done_blocks=[], sync_count=0, sync_gen=0)

    def tma_warp():
        def load(it, buf):
            Q[buf] = it
            bar_q[buf].arrive()                        # complete_tx
        for it in range(min(3, n_iter)):
            load(it, it)
            yield None
        buf, par = 0, 0
        for it in range(n_iter - 3):
            yield (lambda buf=buf, par=par: bar_qfree[buf].passed(par))
            load(it + 3, buf)
            buf += 1
            if buf == 3:
                buf, par = 0, par ^ 1
            yield None

    def scores(it, qb):
        def ex():
            if Q[qb] != it:
                raise Violation(f"score MMA of block {it} read Q/dO of block {Q[qb]}")
            S[it & 1] = it
        return ex

    def dvdk(it, qb):
        def ex():
            if Q[qb] != it:
                raise Violation(f"dV/dK MMA of block {it} read Q/dO of block {Q[qb]}")
            for t in range(n_thr):
                if stage[it & 1][t] != it:
                    raise Violation(f"dV/dK MMA of block {it} read staging written for block {stage[it & 1][t]} (thread {t})")
            state["done_blocks"].append(it)
        return ex

    def mma_warp():
        yield (lambda: bar_q[0].passed(0))
        pipe.issue(scores(0, 0)); pipe.commit(bar_s[0])
        qb, qpar = 0, 0
        for it in range(n_iter):
            nqb, npar = qb + 1, qpar
            if nqb == 3:
                nqb, npar = 0, npar ^ 1
            if it + 1 < n_iter:
                yield (lambda nqb=nqb, npar=npar: bar_q[nqb].passed(npar))
                pipe.issue(scores(it + 1, nqb)); pipe.commit(bar_s[(it + 1) & 1])
            if per_stage_bar_p:
                b, par = bar_p[it & 1], (it >> 1) & 1
            else:
                b, par = bar_p[0], it & 1
            yield (lambda b=b, par=par: b.passed(par))
            pipe.issue(dvdk(it, qb)); pipe.commit(bar_d[it & 1]); pipe.commit(bar_qfree[qb])
            qb, qpar = nqb, npar
            yield None
        state["mma_done"] = True

    def compute(t):
        for it in range(n_iter):
            tb = it & 1
            yield (lambda tb=tb, it=it: bar_s[tb].passed((it >> 1) & 1))
            if S[tb] != it:
                raise Violation(f"thread {t} read scores of block {S[tb]} while working on block {it}")
            if it >= 2:
                yield (lambda tb=tb, it=it: bar_d[tb].passed(((it >> 1) - 1) & 1))
            yield None
            stage[tb][t] = it
            yield None
            (bar_p[tb] if per_stage_bar_p else bar_p[0]).arrive()
            if block_barrier:                            # bwd_compute_bar_sync()
                gen = state["sync_gen"]
                state["sync_count"] += 1
                if state["sync_count"] == n_thr:
                    state["sync_count"], state["sync_gen"] = 0, gen + 1
                yield (lambda gen=gen: state["sync_gen"] != gen)
            else:
                yield None
        yield (lambda: bar_d[(n_iter - 1) & 1].passed(((n_iter - 1) >> 1) & 1))

    agents = {"tma": tma_warp(), "mma": mma_warp(), "pipe": pipe.agent(lambda: state["mma_done"])}
    for t in range(n_thr):
        agents[f"c{t}"] = compute(t)
    res = run(agents, rng)
    if res == "ok" and state["done_blocks"] != list(range(n_iter)):
        raise Violation(f"blocks executed: {state['done_blocks']}")
    return res


# ---------------------------------------------------------------------------------------------
# dQ kernel as it was in builds v3-v8: dS goes to a double-buffered SHARED-MEMORY staging tile, a
# thread waits for bar_dq[tb] (dQ MMA of block j-2 retired) before overwriting it; one bar_p.
# ---------------------------------------------------------------------------------------------
def dq_kernel_v8(njb, rng, n_thr=8):
    pipe = TensorPipe()
    bar_s, bar_dq = [Mbar(1), Mbar(1)], [Mbar(1), Mbar(1)]
    bar_p = Mbar(n_thr)
    S = [None, None]
    stage = [[None] * n_thr for _ in range(2)]
    state = dict(mma_done=False, blocks=[])

    def scores(j):
        def ex():
            S[j & 1] = j
        return ex

    def dq_mma(j):
        def ex():
            for t in range(n_thr):
                if stage[j & 1][t] != j:
                    raise Violation(f"dQ MMA of block {j} read staging written for block {stage[j & 1][t]} (thread {t})")
            state["blocks"].append(j)
        return ex

    def mma_warp():
        pipe.issue(scores(0)); pipe.commit(bar_s[0])
        yield None
        for j in range(njb):
            if j + 1 < njb:
                pipe.issue(scores(j + 1)); pipe.commit(bar_s[(j + 1) & 1])
                yield None
            yield (lambda j=j: bar_p.passed(j & 1))
            pipe.issue(dq_mma(j)); pipe.commit(bar_dq[j & 1])
            yield None
        state["mma_done"] = True

    def compute(t):
        for j in range(njb):
            tb = j & 1
            yield (lambda tb=tb, j=j: bar_s[tb].passed((j >> 1) & 1))
            if S[tb] != j:
                raise Violation(f"thread {t} read scores of block {S[tb]} while working on block {j}")
            if j >= 2:
                yield (lambda tb=tb, j=j: bar_dq[tb].passed(((j >> 1) - 1) & 1))
            yield None
            stage[tb][t] = j
            yield None
            bar_p.arrive()
            yield None
        yield (lambda: bar_dq[(njb - 1) & 1].passed(((njb - 1) >> 1) & 1))

    agents = {"mma": mma_warp(), "pipe": pipe.agent(lambda: state["mma_done"])}
    for t in range(n_thr):
        agents[f"c{t}"] = compute(t)
    res = run(agents, rng)
    if res == "ok" and state["blocks"] != list(range(njb)):
        raise Violation(f"blocks executed: {state['blocks']}")
    return res


# ---------------------------------------------------------------------------------------------
# forward kernel (attn_fwd_kernel): S double-buffered in TMEM, ONE P staging tile and O in TMEM,
# both released by bar_o (PV of the previous block retired); one bar_p. V double-buffered by the
# TMA warp behind bar_vfree (not modelled: it has the dK/dV kernel's Q/dO ring structure).
# ---------------------------------------------------------------------------------------------
def fwd_kernel(njb, rng, n_thr=8, wait_bar_o=True):
    pipe = TensorPipe()
    bar_s = [Mbar(1), Mbar(1)]
    bar_p, bar_o = Mbar(n_thr), Mbar(1)
    S = [None, None]
    P = [None] * n_thr
    state = dict(mma_done=False, blocks=[])

    def scores(j):
        def ex():
            S[j & 1] = j
        return ex

    def pv(j):
        def ex():
            for t in range(n_thr):
                if P[t] != j:
                    raise Violation(f"PV MMA of block {j} read P written for block {P[t]} (thread {t})")
            state["blocks"].append(j)
        return ex

    def mma_warp():
        pipe.issue(scores(0)); pipe.commit(bar_s[0])
        yield None
        for j in range(njb):
            if j + 1 < njb:
                pipe.issue(scores(j + 1)); pipe.commit(bar_s[(j + 1) & 1])
                yield None
            yield (lambda j=j: bar_p.passed(j & 1))
            pipe.issue(pv(j)); pipe.commit(bar_o)
            yield None
        state["mma_done"] = True

    def compute(t):
        for j in range(njb):
            tb = j & 1
            yield (lambda tb=tb, j=j: bar_s[tb].passed((j >> 1) & 1))
            if S[tb] != j:
                raise Violation(f"thread {t} read scores of block {S[tb]} while working on block {j}")
            yield None                                   # softmax math
            if j > 0 and wait_bar_o:
                yield (lambda j=j: bar_o.passed((j - 1) & 1))   # PV(j-1) retired: P tile and O are free
            P[t] = j
            yield None
            bar_p.arrive()
            yield None
        yield (lambda: bar_o.passed((njb - 1) & 1))

    agents = {"mma": mma_warp(), "pipe": pipe.agent(lambda: state["mma_done"])}
    for t in range(n_thr):
        agents[f"c{t}"] = compute(t)
    res = run(agents, rng)
    if res == "ok" and state["blocks"] != list(range(njb)):
        raise Violation(f"blocks executed: {state['blocks']}")
    return res


# ---------------------------------------------------------------------------------------------
# CTA-pair persistent GEMM (gemm.cu gemm_bf16_pair_kernel): TMA producers in both CTAs fill a ring of
# STAGES slots (one full / empty barrier pair per slot, the leader's full barrier collects both CTAs'
# bytes), the leader's MMA warp consumes them into one of two TMEM accumulator stages and commits
# empty (multicast to both CTAs) / tfull (multicast); 4 epilogue warps per CTA drain the
# accumulator and arrive on the LEADER's tempty barrier (count 8).
# ---------------------------------------------------------------------------------------------
def gemm_pair_kernel(num_tiles, num_kb, rng, stages=3, epi_warps=4):
    pipe = TensorPipe()
    full = [Mbar(2) for _ in range(stages)]               # leader's: one complete_tx per CTA (modelled as 2 arrivals)
    empty = [[Mbar(1) for _ in range(stages)] for _ in range(2)]   # per CTA (the commit is multicast)
    tfull = [[Mbar(1), Mbar(1)] for _ in range(2)]        # per CTA (multicast)
    tempty = [Mbar(2 * epi_warps), Mbar(2 * epi_warps)]   # leader's
    slot = [[None] * stages for _ in range(2)]            # per CTA: (tile, kb) whose operand halves are in the slot
    acc = [None, None]                                    # which tile's sum is in accumulator stage a: (tile, kb_count)
    state = dict(mma_done=False, out=[[], []])

    def producer(cta):
        stage, phase = 0, 0
        for tile in range(num_tiles):
            for kb in range(num_kb):
                yield (lambda s=stage, ph=phase: empty[cta][s].passed(ph ^ 1))
                slot[cta][stage] = (tile, kb)
                full[stage].arrive()
                stage += 1
                if stage == stages:
                    stage, phase = 0, phase ^ 1
                yield None

    def mma(tile, kb, stage, a):
        def ex():
            for cta in range(2):
                if slot[cta][stage] != (tile, kb):
                    raise Violation(f"MMA of tile {tile} k-block {kb} read slot holding {slot[cta][stage]} (CTA {cta})")
            if kb == 0:
                acc[a] = [tile, 1]
            else:
                if acc[a][0] != tile:
                    raise Violation(f"MMA of tile {tile} accumulated onto tile {acc[a][0]}")
                acc[a][1] += 1
        return ex

    def commit_multicast(bars):
        def ex():
            for b in bars:
                b.arrive()
        return ex

    def mma_warp():
        stage, phase, a, aph = 0, 0, 0, 0
        for tile in range(num_tiles):
            yield (lambda a=a, aph=aph: tempty[a].passed(aph ^ 1))
            for kb in range(num_kb):
                yield (lambda s=stage, ph=phase: full[s].passed(ph))
                pipe.issue(mma(tile, kb, stage, a))
                pipe.issue(commit_multicast([empty[0][stage], empty[1][stage]]))
                stage += 1
                if stage == stages:
                    stage, phase = 0, phase ^ 1
                yield None
            pipe.issue(commit_multicast([tfull[0][a], tfull[1][a]]))
            a += 1
            if a == 2:
                a, aph = 0, aph ^ 1
            yield None
        state["mma_done"] = True

    def epilogue(cta, w):
        a, aph = 0, 0
        for tile in range(num_tiles):
            yield (lambda a=a, aph=aph: tfull[cta][a].passed(aph))
            if acc[a] != [tile, num_kb]:
                raise Violation(f"epilogue of tile {tile} read accumulator holding {acc[a]}")
            yield None                                   # tcgen05.ld + stores
            if w == 0:
                state["out"][cta].append(tile)
            tempty[a].arrive()
            a += 1
            if a == 2:
                a, aph = 0, aph ^ 1
            yield None

    agents = {"mma": mma_warp(), "pipe": pipe.agent(lambda: state["mma_done"]), "tma0": producer(0), "tma1": producer(1)}
    for cta in range(2):
        for w in range(epi_warps):
            agents[f"epi{cta}{w}"] = epilogue(cta, w)
    res = run(agents, rng)
    if res == "ok" and state["out"] != [list(range(num_tiles))] * 2:
        raise Violation(f"tiles written: {state['out']}")
    return res


# ---------------------------------------------------------------------------------------------
# The sm_90a kernels (gemm.cu, attention.cu): every operand ring is the same protocol. A TMA producer
# thread fills slot i % depth for item i once the slot's FREE barrier has completed the phase of item
# i - depth; TMA copies land asynchronously and in any order, each completing its bytes on the slot's
# FULL barrier; consumer warps wait on FULL, read the slot with wgmma and arrive on FREE once those
# MMAs have retired. Modelled:
#   * `lag` = 1: the GEMM consumers free slot i - 1 only after issuing item i (wgmma.wait_group 1);
#   * `skip(g, i)`: warpgroup g does not read item i (the forward's key block above a warpgroup's diagonal, the dQ
#     kernel's blocks past a warpgroup's last row) but still waits on its FULL barrier before releasing it. The
#     model found why (`skip_waits_full=False`): the warps of a warpgroup are scheduled independently, and a warp
#     that frees a skipped item at once can complete the FREE phase of the item before it in the same slot while
#     another warp still reads that item -- the producer then overwrites it, or a phase is left short for ever;
#   * `ctas` = 2: the cluster GEMM -- each CTA's producer multicasts its half of the slot into both
#     CTAs, and (`remote_release`) every consumer warp arrives on FREE in both CTAs.
# A copy landing in a slot that a consumer is still reading, or a consumer finding a half that does not
# belong to its item, is a Violation.
# ---------------------------------------------------------------------------------------------
def wg_ring_kernel(n_items, depth, rng, ctas=1, warpgroups=2, warps=2, lag=0, skip=None, wait_free=True,
                   remote_release=True, skip_waits_full=True, release_early=False):
    skip = skip or (lambda g, i: False)
    n_cons = warpgroups * warps
    full = [[Mbar(ctas) for _ in range(depth)] for _ in range(ctas)]      # one completion per landed half
    free = [[Mbar(n_cons * (ctas if remote_release else 1)) for _ in range(depth)] for _ in range(ctas)]
    slot = [[[None] * ctas for _ in range(depth)] for _ in range(ctas)]   # [cta][slot][half] = item
    reading = [[set() for _ in range(depth)] for _ in range(ctas)]
    inflight = []                                                          # issued, not yet landed copies
    state = dict(producers=ctas, read=[[[] for _ in range(n_cons)] for _ in range(ctas)])

    def producer(r):
        for i in range(n_items):
            b = i % depth
            if i >= depth and wait_free:
                yield (lambda b=b, i=i: free[r][b].passed(((i // depth) - 1) & 1))
            for dst in range(ctas):                                        # multicast: the same half into every CTA
                inflight.append((dst, b, r, i))
            yield None
        state["producers"] -= 1

    def dma():
        while True:
            if inflight:
                dst, b, half, i = inflight.pop(rng.randrange(len(inflight)))
                if reading[dst][b]:
                    raise Violation(f"copy of item {i} landed in CTA {dst} slot {b} while {sorted(reading[dst][b])} read it")
                slot[dst][b][half] = i
                full[dst][b].arrive()
                yield None
            elif state["producers"] == 0:
                return
            else:
                yield (lambda: bool(inflight) or state["producers"] == 0)

    def release(c, b):
        free[c][b].arrive()
        if ctas == 2 and remote_release:
            free[c ^ 1][b].arrive()

    def consumer(c, g, w):
        me = (c, g, w)
        prev = None
        for i in range(n_items):
            b = i % depth
            if skip(g, i):
                if skip_waits_full:
                    yield (lambda b=b, i=i: full[c][b].passed((i // depth) & 1))
                release(c, b)
                yield None
                continue
            yield (lambda b=b, i=i: full[c][b].passed((i // depth) & 1))
            reading[c][b].add(me)
            if slot[c][b] != [i] * ctas:
                raise Violation(f"consumer {me} found {slot[c][b]} in slot {b} while on item {i} (stale)")
            state["read"][c][g * warps + w].append(i)
            yield None                                                     # the MMAs read the slot
            if release_early:                                              # freed at issue, not once they retired
                release(c, b)
            if lag and prev is not None:
                reading[c][prev].discard(me)
                if not release_early:
                    release(c, prev)
            if lag:
                prev = b
            else:
                reading[c][b].discard(me)
                release(c, b)
            yield None
        if prev is not None:
            reading[c][prev].discard(me)
            if not release_early:
                release(c, prev)

    agents = {"dma": dma()}
    for r in range(ctas):
        agents[f"tma{r}"] = producer(r)
        for g in range(warpgroups):
            for w in range(warps):
                agents[f"c{r}{g}{w}"] = consumer(r, g, w)
    res = run(agents, rng)
    if res == "ok":
        for c in range(ctas):
            for g in range(warpgroups):
                want = [i for i in range(n_items) if not skip(g, i)]
                for w in range(warps):
                    if state["read"][c][g * warps + w] != want:
                        raise Violation(f"consumer {(c, g, w)} read items {state['read'][c][g * warps + w]}")
    return res


def wg_fwd_kernel(njb, rng, **kw):
    """attn_fwd_kernel's K ring and V ring (2 slots each): warpgroup 0 skips the last key block, which lies above
    its diagonal"""
    return wg_ring_kernel(njb, 2, rng, skip=lambda g, j: g == 0 and j == njb - 1, **kw)


def wg_dq_kernel(njb, rng, **kw):
    """attn_bwd_dq_kernel's K/V ring (3 slots): warpgroup g skips the key blocks past njb - 2 + g"""
    return wg_ring_kernel(njb, 3, rng, skip=lambda g, j: j > njb - 2 + g, **kw)


def wg_dkdv_kernel(n_iter, rng, **kw):
    """attn_bwd_dkdv_kernel's Q/dO ring (3 slots): every warpgroup waits on every block (its 16-query slices
    before its keys are skipped after the wait)"""
    return wg_ring_kernel(n_iter, 3, rng, **kw)


# The pipelined attention rings: a warpgroup leaves block i's accumulating product (P V, dV / dK, dQ) in flight while
# block i + 1's scores run, and frees the buffer that product reads one block late (lag 1). `release_early` frees it
# at issue instead, the hazard the lag exists for.
def wg_fwd_v_kernel(njb, rng, **kw):
    """attn_fwd_kernel's V ring (2 slots, lag 1; its K ring is wg_fwd_kernel's): warpgroup 0 skips the last key
    block after waiting for its loads"""
    return wg_ring_kernel(njb, 2, rng, lag=1, skip=lambda g, j: g == 0 and j == njb - 1, **kw)


def wg_dq_lag_kernel(njb, rng, **kw):
    """attn_bwd_dq_kernel's K/V ring (4 slots, lag 1): warpgroup g skips the key blocks past njb - 2 + g"""
    return wg_ring_kernel(njb, 4, rng, lag=1, skip=lambda g, j: j > njb - 2 + g, **kw)


def wg_dkdv_lag_kernel(n_iter, rng, **kw):
    """attn_bwd_dkdv_kernel's Q/dO ring (4 slots, lag 1): every warpgroup computes every block"""
    return wg_ring_kernel(n_iter, 4, rng, lag=1, **kw)


def wg_gemm_kernel(num_items, rng, stages=4, ctas=1, **kw):
    """gemm_bf16_kernel (ctas = 1) and gemm_bf16_pair_kernel (ctas = 2): the operand ring over all k-blocks of
    all tiles of a CTA, each slot freed one k-block late"""
    return wg_ring_kernel(num_items, stages, rng, ctas=ctas, lag=1, **kw)


def explore(kernel, trials, seed=0, **kw):
    """-> (#ok, first violation or None, other outcomes)"""
    ok, first, other = 0, None, {}
    for i in range(trials):
        rng = random.Random(seed * 100003 + i)
        try:
            r = kernel(rng=rng, **kw)
        except Violation as v:
            first = first or f"trial {i}: {v}"
            continue
        if r == "ok":
            ok += 1
        else:
            other[r] = other.get(r, 0) + 1
    return ok, first, other


if __name__ == "__main__":
    for name, fn, kw in [("dQ v9 (one bar_p)", dq_kernel, dict(njb=8, per_stage_bar_p=False)),
                         ("dQ v10 (bar_p per stage)", dq_kernel, dict(njb=8, per_stage_bar_p=True)),
                         ("dQ v3-v8 (smem staging, one bar_p)", dq_kernel_v8, dict(njb=8)),
                         ("forward shipped", fwd_kernel, dict(njb=8)),
                         ("forward without the bar_o wait", fwd_kernel, dict(njb=8, wait_bar_o=False)),
                         ("dK/dV shipped (one bar_p)", dkdv_kernel, dict(n_iter=2)),
                         ("dK/dV with bar_p per stage", dkdv_kernel, dict(n_iter=2, per_stage_bar_p=True)),
                         ("dK/dV per stage, no block barrier", dkdv_kernel, dict(n_iter=9, per_stage_bar_p=True, block_barrier=False)),
                         ("dK/dV without the block barrier", dkdv_kernel, dict(n_iter=9, block_barrier=False)),
                         ("pair GEMM, 5 tiles x 7 k-blocks", gemm_pair_kernel, dict(num_tiles=5, num_kb=7)),
                         ("pair GEMM, 1 tile x 1 k-block", gemm_pair_kernel, dict(num_tiles=1, num_kb=1)),
                         ("sm_90a forward", wg_fwd_kernel, dict(njb=8)),
                         ("sm_90a dQ", wg_dq_kernel, dict(njb=8)),
                         ("sm_90a dK/dV", wg_dkdv_kernel, dict(n_iter=9)),
                         ("sm_90a cluster GEMM", wg_gemm_kernel, dict(num_items=13, ctas=2)),
                         ("sm_90a cluster GEMM, local release", wg_gemm_kernel, dict(num_items=13, ctas=2, remote_release=False))]:
        ok, first, other = explore(fn, 2000, **kw)
        print(f"{name:36s} ok {ok:4d}/2000   first violation: {first}   other: {other}")
