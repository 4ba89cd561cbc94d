"""Discrete-event model of a warp-specialised fused tensor-core layer schedule for single-thread-issued MMAs whose
completion is committed to mbarriers (the tcgen05 model of issue; csrc/wn_tc_kernel.cu issues wgmma from its consumer
warpgroups instead and does not use this schedule): producer warp, issuer roles A / B, history-copy role C and the
eight epilogue warps exchange mbarrier phases, weight-ring stages and MMA commits, with randomised latencies.  It checks what cannot be seen in a passing GPU run:

  * deadlock: every role must finish every sample;
  * phase aliasing: an mbarrier waiter may never be two completed phases behind (parity waits would then block
    for ever or pass early) -- the model tracks, per waiter, WHICH completion it is waiting for;
  * late commits: a commit issued when its thread has no MMA in flight never arrives;
  * ring order: every role consumes the chunk the producer put into that stage;
  * the data hazards the handshakes exist for (h / x tiles, accumulators, conditioning buffers).

Pure Python, no GPU.  `python tools/tc_protocol_model.py [runs]` runs random trials; tests/test_tc_protocol_model.py
runs a bounded number of them.
"""
import heapq
import random
import sys


class Hazard(Exception):
    pass


class Barrier:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.completed = name, count, count, 0
        self.waiters = []                                        # (role, generator, k): blocked on completion number k
        self.sim = None

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.completed += 1
            self.pending = self.count
            still = []
            for name, gen, k in self.waiters:
                if self.completed == k + 1:
                    self.sim.waiting.pop(name, None)
                    self.sim._push(self.sim.now + self.sim.lat(name, 60, 250), name, gen)      # wake-up latency of a parked try_wait
                elif self.completed > k + 1:
                    raise Hazard(f"{name}: {self.name} completed {self.completed} times while it waits for completion #{k} (phase aliasing)")
                else:
                    still.append((name, gen, k))
            self.waiters = still


class Sim:
    def __init__(self, L=20, S=256, nstage=6, NC=2, steps=3, dil=None, dump_last=False, t0=0, seed=0, slow=None, bug=None):
        self.L, self.SKC, self.nstage, self.NC, self.steps, self.t0 = L, S // 128, nstage, NC, steps, t0
        self.KT = (S // 64, 4)                                   # k-tiles of the two output GEMMs (A = 256)
        self.dil = dil or [1 << (i % 10) for i in range(L)]
        self.dump_last = dump_last
        self.rng = random.Random(seed)
        self.slow = slow or {}                                   # role name -> latency multiplier (stress a role)
        self.bug = bug                                           # re-introduce a defect the hardware runs hit (the model must see it)
        self.now = 0
        self.q = []
        self.seq = 0
        self.NE = 8                                              # epilogue warps (each arrives once per phase in the model)
        B = lambda n, c=1: Barrier(n, c)
        self.w_full = [B(f"w_full{s}") for s in range(nstage)]
        self.w_empty = [B(f"w_empty{s}") for s in range(nstage)]
        self.epi_done = [B("epi_done0", self.NE), B("epi_done1", self.NE)]   # alternate by publication number
        self.d1_full, self.dx_full = B("d1_full"), B("dx_full")
        self.skip_full, self.out_full = B("skip_full", 2), B("out_full", 2)
        self.pre_done = B("pre_done", self.NE)
        self.cond_full = [B(f"cond_full{i}") for i in range(NC)]
        self.cond_empty = [B(f"cond_empty{i}", self.NE) for i in range(NC)]
        self.cx_done = B("cx_done")
        self.b_done = [B("b_done0"), B("b_done1")]
        self.hx_full = B("hx_full", self.NE)
        self.hx_done = [B("hx_done0"), B("hx_done1")]
        self.stage_content = [None] * nstage                    # what the producer put there (checked by consumers)
        self.mma_busy_until = 0                                  # the tensor pipe executes in issue order
        self.inflight = {}                                       # thread -> completion time of its latest MMA
        self.waiting = {}                                        # role -> description (for deadlock reports)
        self.finished = set()
        self.late_commits = []
        # data-hazard bookkeeping: resource -> (readers_done_time, last_write_time)
        self.res_read_until = {}
        self.log = []

    # ------------------------------------------------------------------ engine
    def lat(self, role, lo, hi):
        return int(self.rng.uniform(lo, hi) * self.slow.get(role.split("#")[0], 1.0))

    def spawn(self, name, gen):
        self._push(self.now, name, gen)

    def _push(self, t, name, gen):
        self.seq += 1
        heapq.heappush(self.q, (t, self.seq, name, gen))

    def run(self, limit=10**9):
        roles = set()
        while self.q:
            t, _, name, gen = heapq.heappop(self.q)
            roles.add(name)
            self.now = max(self.now, t)
            if self.now > limit:
                raise Hazard("time limit")
            try:
                req = next(gen)
            except StopIteration:
                self.finished.add(name)
                self.waiting.pop(name, None)
                continue
            kind = req[0]
            if kind == "delay":
                self._push(self.now + req[1], name, gen)
            elif kind == "wait":                                 # ("wait", barrier, k): completion number k (0-based)
                _, bar, k = req
                if bar.completed > k + 1:
                    raise Hazard(f"{name}: {bar.name} completed {bar.completed} times while waiting for completion #{k} (phase aliasing)")
                if bar.completed == k + 1:
                    self.waiting.pop(name, None)
                    self._push(self.now + self.lat(name, 20, 120), name, gen)
                else:
                    bar.sim = self
                    self.waiting[name] = f"{bar.name} #{k}"
                    bar.waiters.append((name, gen, k))
            else:
                raise AssertionError(kind)
        missing = roles - self.finished - {"_event"}
        if missing:
            raise Hazard("deadlock: " + "; ".join(f"{r} waits for {self.waiting.get(r)}" for r in sorted(missing)))

    # ------------------------------------------------------------------ tcgen05 / TMA primitives
    def mma(self, thread, n_instr, reads=(), writes=()):
        """n_instr MMAs from `thread`, the last one issued NOW (callers delay for the issue time first); returns the
        completion time.  Pipeline latency >= 100 cycles after the last issue, 64 cycles per N=128 instruction."""
        start = max(self.now + 100 - 45 * (n_instr - 1), self.mma_busy_until)
        done = start + 64 * n_instr
        self.mma_busy_until = done
        self.inflight[thread] = done
        for r in reads:
            self.res_read_until[r] = max(self.res_read_until.get(r, 0), done)
        for w in writes:
            self.res_read_until[("w",) + tuple([w])] = max(self.res_read_until.get(("w", w), 0), done)
        return done

    def commit(self, thread, bar, what):
        done = self.inflight.get(thread, 0)
        if done <= self.now:
            self.late_commits.append((thread, what, self.now))
            raise Hazard(f"{thread}: tcgen05.commit({what}) issued with no MMA of this thread in flight")
        self.at(done + 30, bar.arrive)

    def at(self, t, fn):
        def g():
            fn()
            return
            yield
        self._push(t, "_event", _once(fn))

    def write_ok(self, role, res):
        if self.res_read_until.get(res, 0) > self.now:
            raise Hazard(f"{role}: writes {res} while an MMA / copy still reads it")

    def mma_write_ok(self, role, res):
        pass


def _once(fn):
    fn()
    return
    yield


# ---------------------------------------------------------------------- the roles
def build(sim):
    L, SKC, nstage, NC = sim.L, sim.SKC, sim.nstage, sim.NC
    dil = sim.dil
    T = range(sim.t0, sim.t0 + sim.steps)
    dstep_of = lambda t: sim.dump_last and t == sim.t0 + sim.steps - 1

    def chunk_sequence(t):
        """ring chunks of one sample in producer order: (owner, tag)"""
        ds = dstep_of(t)
        seq = []
        if t >= 1: seq += [("A", ("pa", 0)), ("A", ("pw", 0))]
        seq.append(("A", ("cur", 0)))
        if L > 1:
            if t >= dil[1]: seq += [("B", ("pa", 1)), ("B", ("pw", 1))]
            seq.append(("A", ("cur", 1)))
        for l in range(1, L):
            seq.append(("A", ("res", l - 1)))
            sk = [(("A" if ds else "B"), ("skip", l - 1, c)) for c in range(SKC)]
            if ds: seq += sk
            seq.append(("A", ("wf", l)))
            if not ds: seq += sk
            if l + 1 < L:
                if t >= dil[l + 1]: seq += [("B", ("pa", l + 1)), ("B", ("pw", l + 1))]
                seq.append(("A", ("cur", l + 1)))
        if ds: seq.append(("A", ("res", L - 1)))
        seq += [(("A" if ds else "B"), ("skip", L - 1, c)) for c in range(SKC)]
        for g in range(2):
            for kt in range(sim.KT[g]):
                seq += [("A", ("out", g, kt, 0)), ("B", ("out", g, kt, 1))]
        return seq

    # ---------------- producer
    def producer():
        stage, lap = 0, 0
        g_cond = 0
        for t in T:
            ds = dstep_of(t)
            ring = iter(chunk_sequence(t))

            def put(expect_tag):
                nonlocal stage, lap
                owner, tag = next(ring)
                assert tag[:len(expect_tag)] == expect_tag, (tag, expect_tag)
                if lap > 0:
                    yield ("wait", sim.w_empty[stage], lap - 1)
                s = stage
                def land(s=s, tag=tag):
                    sim.stage_content[s] = tag
                    sim.w_full[s].arrive()
                sim.at(sim.now + sim.lat("P", 300, 1200), land)
                stage += 1
                if stage == nstage: stage, lap = 0, lap + 1
                yield ("delay", sim.lat("P", 30, 80))

            def put_cond(l):
                nonlocal g_cond
                cb, k = g_cond % NC, g_cond // NC
                if k > 0:
                    yield ("wait", sim.cond_empty[cb], k - 1)
                sim.at(sim.now + sim.lat("P", 400, 1500), sim.cond_full[cb].arrive)
                g_cond += 1
                yield ("delay", 40)

            def put_prev(l):
                if t >= dil[l]:
                    yield from put(("pa", l)); yield from put(("pw", l))

            yield from put_cond(0)
            yield from put_prev(0)
            yield from put(("cur", 0))
            if L > 1:
                yield from put_cond(1)
                yield from put_prev(1)
                yield from put(("cur", 1))
            for l in range(1, L):
                if (NC == 2 or sim.bug == 'cond_first') and l + 1 < L: yield from put_cond(l + 1)
                yield from put(("res", l - 1))
                if ds:
                    for c in range(SKC): yield from put(("skip", l - 1))
                yield from put(("wf", l))
                if not ds:
                    for c in range(SKC): yield from put(("skip", l - 1))
                if l + 1 < L:
                    if NC == 1 and sim.bug != 'cond_first': yield from put_cond(l + 1)
                    yield from put_prev(l + 1)
                    yield from put(("cur", l + 1))
            if ds: yield from put(("res", L - 1))
            for c in range(SKC): yield from put(("skip", L - 1))
            for g in range(2):
                for kt in range(sim.KT[g]):
                    yield from put(("out", g, kt, 0)); yield from put(("out", g, kt, 1))

    # ---------------- common consumer helpers
    class Walker:
        def __init__(self, who):
            self.who, self.stage, self.lap = who, 0, 0
        def advance(self):
            self.stage += 1
            if self.stage == nstage: self.stage, self.lap = 0, self.lap + 1
        def skipc(self, n):
            for _ in range(n): self.advance()
        def take(self, tag):
            """wait_stage: returns the stage index once the chunk landed; checks it is the expected chunk"""
            yield ("wait", sim.w_full[self.stage], self.lap)
            got = sim.stage_content[self.stage]
            if got[:len(tag)] != tag:
                raise Hazard(f"{self.who}: expected chunk {tag} in stage {self.stage}, found {got}")
            return self.stage

    def issuer_A():
        w = Walker("A")
        k_epi = k_pre = 0
        k_hx = [0, 0]
        for t in T:
            ds = dstep_of(t)
            yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1                                  # x_0
            if t >= 1:
                sa = yield from w.take(("pa", 0)); w.advance()
                sb = yield from w.take(("pw", 0))
                yield ("delay", sim.lat("A", 150, 300))
                sim.mma("A", 4, reads=[("ring", sa), ("ring", sb)])
                sim.commit("A", sim.w_empty[sa], "w_empty"); sim.commit("A", sim.w_empty[sb], "w_empty"); w.advance()
                yield ("delay", sim.lat("A", 40, 100))
            s = yield from w.take(("cur", 0))
            yield ("delay", sim.lat("A", 150, 300))
            sim.mma("A", 4, reads=[("X", 0), ("ring", s)])
            sim.commit("A", sim.d1_full, "d1_full"); sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
            yield ("delay", sim.lat("A", 40, 100))
            if L > 1:
                hp = t >= dil[1]
                if hp: w.skipc(2)
                s = yield from w.take(("cur", 1))
                yield ("delay", sim.lat("A", 150, 300))
                sim.mma("A", 4, reads=[("X", 0), ("ring", s)])
                if hp: sim.commit("A", sim.cx_done, "cx_done")
                sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
                yield ("delay", sim.lat("A", 40, 100))
            for l in range(1, L):
                hpn = (l + 1 < L) and t >= dil[l + 1]
                s = yield from w.take(("res", l - 1))
                if not ds:
                    s1 = 0 if w.stage + 1 == nstage else w.stage + 1
                    yield ("wait", sim.w_full[s1], w.lap + (1 if s1 == 0 else 0))
                yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1                              # h_{l-1}
                yield ("delay", sim.lat("A", 120, 250))
                sim.mma("A", 4, reads=[("H", (l - 1) & 1), ("ring", s)])
                sim.commit("A", sim.dx_full, "dx_full"); sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
                yield ("delay", sim.lat("A", 50, 120))
                if ds:
                    sts = []
                    for c in range(SKC):
                        sts.append((yield from w.take(("skip", l - 1)))); w.advance()
                    yield ("delay", sim.lat("A", 300, 600))
                    sim.mma("A", 4 * SKC, reads=[("H", (l - 1) & 1)] + [("ring", x) for x in sts])
                    for x in sts: sim.commit("A", sim.w_empty[x], "w_empty")
                    yield ("delay", sim.lat("A", 40, 100))
                s = yield from w.take(("wf", l))
                yield ("delay", sim.lat("A", 120, 250))
                sim.mma("A", 4, reads=[("H", (l - 1) & 1), ("ring", s)])
                sim.commit("A", sim.d1_full, "d1_full"); sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
                yield ("delay", sim.lat("A", 50, 120))
                if not ds: w.skipc(SKC)
                yield ("wait", sim.hx_done[(l - 1) & 1], k_hx[(l - 1) & 1]); k_hx[(l - 1) & 1] += 1
                yield ("wait", sim.pre_done, k_pre); k_pre += 1
                if l + 1 < L:
                    if hpn: w.skipc(2)
                    s = yield from w.take(("cur", l + 1))
                    yield ("delay", sim.lat("A", 150, 300))
                    sim.mma("A", 4, reads=[("X", l & 1), ("ring", s)])
                    if hpn: sim.commit("A", sim.cx_done, "cx_done")
                    sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
                    yield ("delay", sim.lat("A", 40, 100))
            yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1                                  # h_{L-1}
            yield ("wait", sim.hx_done[(L - 1) & 1], k_hx[(L - 1) & 1]); k_hx[(L - 1) & 1] += 1
            if ds:
                s = yield from w.take(("res", L - 1))
                yield ("delay", sim.lat("A", 150, 300))
                sim.mma("A", 4, reads=[("H", (L - 1) & 1), ("ring", s)])
                sim.commit("A", sim.dx_full, "dx_full"); sim.commit("A", sim.w_empty[s], "w_empty"); w.advance()
                sts = []
                for c in range(SKC):
                    sts.append((yield from w.take(("skip", L - 1)))); w.advance()
                yield ("delay", sim.lat("A", 300, 600))
                sim.mma("A", 4 * SKC, reads=[("H", (L - 1) & 1)] + [("ring", x) for x in sts])
                for x in sts: sim.commit("A", sim.w_empty[x], "w_empty")
                sim.commit("A", sim.skip_full, "skip_full")
            else:
                w.skipc(SKC)
            sim.skip_full.arrive()
            for g in range(2):
                yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1                              # skq / zsq
                for kt in range(sim.KT[g]):
                    s = yield from w.take(("out", g, kt, 0))
                    yield ("delay", sim.lat("A", 150, 300))
                    sim.mma("A", 4, reads=[("BIG", kt), ("ring", s)])
                    sim.commit("A", sim.w_empty[s], "w_empty")
                    if kt == sim.KT[g] - 1: sim.commit("A", sim.out_full, "out_full")
                    w.advance(); w.skipc(1)
                    yield ("delay", sim.lat("A", 40, 100))

    def issuer_B():
        w = Walker("B")
        k_epi = k_cx = 0
        for t in T:
            ds = dstep_of(t)

            def prev_b(l, done_bar):
                nonlocal k_cx
                yield ("wait", sim.cx_done, k_cx); k_cx += 1
                sa = yield from w.take(("pa", l)); w.advance()
                sb = yield from w.take(("pw", l))
                yield ("delay", sim.lat("B", 150, 300))
                sim.mma("B", 4, reads=[("ring", sa), ("ring", sb)])
                sim.commit("B", sim.w_empty[sa], "w_empty"); sim.commit("B", sim.w_empty[sb], "w_empty"); w.advance()
                if done_bar is not None: sim.commit("B", done_bar, done_bar.name)
                yield ("delay", sim.lat("B", 40, 100))

            def skip_layer(l, done_bar):
                sts = []
                for c in range(SKC):
                    sts.append((yield from w.take(("skip", l)))); w.advance()
                yield ("delay", sim.lat("B", 300, 600))
                sim.mma("B", 4 * SKC, reads=[("H", l & 1)] + [("ring", x) for x in sts])
                for x in sts: sim.commit("B", sim.w_empty[x], "w_empty")
                if done_bar is not None: sim.commit("B", done_bar, done_bar.name)
                yield ("delay", sim.lat("B", 40, 100))

            bsig = lambda j: sim.b_done[0 if sim.bug == 'one_b_done' else (j & 1)]

            yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1
            if t >= 1: w.skipc(2)
            w.skipc(1)
            if L > 1:
                if t >= dil[1]: yield from prev_b(1, bsig(0))
                elif sim.bug == 'empty_commit': sim.commit('B', bsig(0), 'b_done')
                else: bsig(0).arrive()
                w.skipc(1)
            for l in range(1, L):
                w.skipc(1)
                yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1
                hpn = (l + 1 < L) and t >= dil[l + 1]
                if ds: w.skipc(SKC + 1)
                else:
                    w.skipc(1)
                    yield from skip_layer(l - 1, None if hpn else bsig(l))
                if l + 1 < L:
                    if hpn: yield from prev_b(l + 1, bsig(l))
                    w.skipc(1)
                if ds and not hpn: bsig(l).arrive()
                yield ("delay", sim.lat("B", 20, 80))
            yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1
            if ds: w.skipc(1 + SKC)
            else: yield from skip_layer(L - 1, sim.skip_full)
            for g in range(2):
                yield ("wait", sim.epi_done[0 if sim.bug == "one_epi_done" else k_epi & 1], k_epi if sim.bug == "one_epi_done" else k_epi // 2); k_epi += 1
                for kt in range(sim.KT[g]):
                    w.skipc(1)
                    s = yield from w.take(("out", g, kt, 1))
                    yield ("delay", sim.lat("B", 150, 300))
                    sim.mma("B", 4, reads=[("BIG", kt), ("ring", s)])
                    sim.commit("B", sim.w_empty[s], "w_empty")
                    if kt == sim.KT[g] - 1: sim.commit("B", sim.out_full, "out_full")
                    w.advance()
                    yield ("delay", sim.lat("B", 40, 100))

    def copier_C():
        k = 0
        for t in T:
            for l in range(L):
                yield ("wait", sim.hx_full, k); k += 1
                # bulk copy reads the x tile until it completes
                dur = sim.lat("C", 400, 1800)
                sim.res_read_until[("X", l & 1)] = max(sim.res_read_until.get(("X", l & 1), 0), sim.now + dur)
                yield ("delay", dur)
                sim.hx_done[l & 1].arrive()

    def epilogue(wi):
        name = f"E#{wi}"
        k_d1 = k_dx = k_skip = k_out = 0
        k_bd = [0, 0]
        g_pre = 0
        n_pub = 0
        def publish():
            nonlocal n_pub
            sim.epi_done[0 if sim.bug == "one_epi_done" else n_pub & 1].arrive(); n_pub += 1
        for t in T:
            ds = dstep_of(t)
            yield ("delay", sim.lat(name, 200, 500))                                      # embedding
            sim.write_ok(name, ("X", 0))
            publish(); sim.hx_full.arrive()
            for l in range(L):
                late_cond = sim.bug == "cond_first"              # the defective version also read the tile after the residual
                if not late_cond:
                    cb, k = g_pre % NC, g_pre // NC
                    yield ("wait", sim.cond_full[cb], k)
                    yield ("delay", sim.lat(name, 100, 300))
                    sim.cond_empty[cb].arrive(); g_pre += 1
                if l > 0:
                    yield ("wait", sim.dx_full, k_dx); k_dx += 1
                    yield ("delay", sim.lat(name, 250, 600))
                    sim.write_ok(name, ("X", l & 1))
                    sim.pre_done.arrive(); sim.hx_full.arrive()
                    bi = 0 if sim.bug == 'one_b_done' else (l - 1) & 1
                    yield ("wait", sim.b_done[bi], k_bd[bi]); k_bd[bi] += 1
                if late_cond:
                    cb, k = g_pre % NC, g_pre // NC
                    yield ("wait", sim.cond_full[cb], k)
                    yield ("delay", sim.lat(name, 100, 300))
                    sim.cond_empty[cb].arrive(); g_pre += 1
                yield ("wait", sim.d1_full, k_d1); k_d1 += 1
                yield ("delay", sim.lat(name, 300, 800))                                  # gate
                sim.write_ok(name, ("H", l & 1))
                publish()
            if L > 1:
                bi = 0 if sim.bug == 'one_b_done' else (L - 1) & 1
                yield ("wait", sim.b_done[bi], k_bd[bi]); k_bd[bi] += 1
            if ds:
                yield ("wait", sim.dx_full, k_dx); k_dx += 1
                yield ("delay", sim.lat(name, 200, 400))
            yield ("wait", sim.skip_full, k_skip); k_skip += 1
            yield ("delay", sim.lat(name, 800, 1600))
            for r in [("X", 0), ("X", 1), ("H", 0), ("H", 1)]: sim.write_ok(name, r)
            publish()                                                                      # skq
            yield ("wait", sim.out_full, k_out); k_out += 1
            yield ("delay", sim.lat(name, 800, 1600))
            for kt in range(4): sim.write_ok(name, ("BIG", kt))
            publish()                                                                      # zsq
            yield ("wait", sim.out_full, k_out); k_out += 1
            yield ("delay", sim.lat(name, 2000, 4000))                                    # softmax + sample

    sim.spawn("P", producer())
    sim.spawn("A", issuer_A())
    sim.spawn("B", issuer_B())
    sim.spawn("C", copier_C())
    for wi in range(sim.NE):
        sim.spawn(f"E#{wi}", epilogue(wi))


def build_unfused(sim):
    """The two-round-trip schedule (single issuer, conditioning pre-stored into the accumulator by the epilogue):
    what launches that fill the GPU use.  skip_full / out_full have ONE arrival here."""
    L, SKC, nstage, NC = sim.L, sim.SKC, sim.nstage, sim.NC
    dil = sim.dil
    T = range(sim.t0, sim.t0 + sim.steps)
    sim.skip_full.count = sim.skip_full.pending = 1
    sim.out_full.count = sim.out_full.pending = 1

    def producer():
        stage, lap, g_cond = 0, 0, 0
        for t in T:
            def put(tag):
                nonlocal stage, lap
                if lap > 0:
                    yield ("wait", sim.w_empty[stage], lap - 1)
                s = stage
                def land(s=s, tag=tag):
                    sim.stage_content[s] = tag
                    sim.w_full[s].arrive()
                sim.at(sim.now + sim.lat("P", 300, 1200), land)
                stage += 1
                if stage == nstage: stage, lap = 0, lap + 1
                yield ("delay", sim.lat("P", 30, 80))
            def put_cond():
                nonlocal g_cond
                cb, k = g_cond % NC, g_cond // NC
                if k > 0:
                    yield ("wait", sim.cond_empty[cb], k - 1)
                sim.at(sim.now + sim.lat("P", 400, 1500), sim.cond_full[cb].arrive)
                g_cond += 1
                yield ("delay", 40)
            def put_prev(l):
                if t >= dil[l]:
                    yield from put(("pa", l)); yield from put(("pw", l))
            yield from put_cond()
            yield from put_prev(0)
            for l in range(L):
                if l + 1 < L: yield from put_cond()
                yield from put(("cur", l))
                if l > 0:
                    for c in range(SKC): yield from put(("skip", l - 1, c))
                yield from put(("res", l))
                if l + 1 < L: yield from put_prev(l + 1)
            for c in range(SKC): yield from put(("skip", L - 1, c))
            for g in range(2):
                for kt in range(sim.KT[g]):
                    for nh in range(2): yield from put(("out", g, kt, nh))

    def issuer():
        stage, lap = 0, 0
        k_epi = k_pre = 0
        def take(tag):
            nonlocal stage, lap
            yield ("wait", sim.w_full[stage], lap)
            got = sim.stage_content[stage]
            if got[:len(tag)] != tag:
                raise Hazard(f"issuer: expected chunk {tag} in stage {stage}, found {got}")
            s = stage
            stage += 1
            if stage == nstage: stage, lap = 0, lap + 1
            return s
        def wait_epi():
            nonlocal k_epi
            yield ("wait", sim.epi_done[k_epi & 1], k_epi // 2); k_epi += 1
        def group(n, reads, bars):
            yield ("delay", sim.lat("A", 150, 300))
            sim.mma("A", n, reads=reads)
            for b in bars: sim.commit("A", b, b.name)
            yield ("delay", sim.lat("A", 40, 100))
        def open_layer(l, has_prev):
            nonlocal k_pre
            yield ("wait", sim.pre_done, k_pre); k_pre += 1
            if has_prev:
                sa = yield from take(("pa", l)); sb = yield from take(("pw", l))
                yield from group(4, [("ring", sa), ("ring", sb)], [sim.w_empty[sa], sim.w_empty[sb]])
        def skip_layer(l, done):
            sts = []
            for c in range(SKC): sts.append((yield from take(("skip", l, c))))
            yield from group(4 * SKC, [("H", l & 1)] + [("ring", x) for x in sts], [sim.w_empty[x] for x in sts] + ([done] if done else []))
        for t in T:
            for l in range(L):
                s = None
                if l > 0: s = yield from take(("cur", l))
                yield from wait_epi()                                   # x_l
                if l == 0:
                    yield from open_layer(0, t >= 1)
                    s = yield from take(("cur", 0))
                yield from group(4, [("X", 0), ("ring", s)], [sim.d1_full, sim.w_empty[s]])
                if l > 0: yield from skip_layer(l - 1, None)
                s = yield from take(("res", l))
                yield from wait_epi()                                   # h_l
                yield from group(4, [("H", l & 1), ("ring", s)], [sim.dx_full, sim.w_empty[s]])
                if l + 1 < L: yield from open_layer(l + 1, t >= dil[l + 1])
            yield from skip_layer(L - 1, sim.skip_full)
            for g in range(2):
                yield from wait_epi()
                for kt in range(sim.KT[g]):
                    for nh in range(2):
                        s = yield from take(("out", g, kt, nh))
                        last = kt == sim.KT[g] - 1 and nh == 1
                        yield from group(4, [("BIG", kt), ("ring", s)], [sim.w_empty[s]] + ([sim.out_full] if last else []))

    def epilogue(wi):
        name = f"E#{wi}"
        k_d1 = k_dx = k_skip = k_out = 0
        g_pre = n_pub = 0
        def publish():
            nonlocal n_pub
            sim.epi_done[n_pub & 1].arrive(); n_pub += 1
        def prestore():
            nonlocal g_pre
            cb, k = g_pre % NC, g_pre // NC
            yield ("wait", sim.cond_full[cb], k)
            yield ("delay", sim.lat(name, 150, 500))
            sim.cond_empty[cb].arrive(); sim.pre_done.arrive(); g_pre += 1
        for t in T:
            yield from prestore()
            yield ("delay", sim.lat(name, 200, 500))                    # embedding
            sim.write_ok(name, ("X", 0)); publish()
            for l in range(L):
                yield ("wait", sim.d1_full, k_d1); k_d1 += 1
                yield ("delay", sim.lat(name, 300, 800))
                sim.write_ok(name, ("H", l & 1)); publish()             # h_l
                if l + 1 < L: yield from prestore()
                yield ("wait", sim.dx_full, k_dx); k_dx += 1
                yield ("delay", sim.lat(name, 250, 600))
                if l + 1 < L:
                    sim.write_ok(name, ("X", 0)); publish()             # x_{l+1}
            yield ("wait", sim.skip_full, k_skip); k_skip += 1
            yield ("delay", sim.lat(name, 800, 1600))
            for r in [("X", 0), ("H", 0), ("H", 1)]: sim.write_ok(name, r)
            publish()
            yield ("wait", sim.out_full, k_out); k_out += 1
            yield ("delay", sim.lat(name, 800, 1600))
            for kt in range(4): sim.write_ok(name, ("BIG", kt))
            publish()
            yield ("wait", sim.out_full, k_out); k_out += 1
            yield ("delay", sim.lat(name, 2000, 4000))

    sim.spawn("P", producer())
    sim.spawn("A", issuer())
    for wi in range(sim.NE):
        sim.spawn(f"E#{wi}", epilogue(wi))


def trial(seed, schedule="fused", **kw):
    sim = Sim(seed=seed, **kw)
    (build if schedule == "fused" else build_unfused)(sim)
    sim.run()
    return sim


def main(runs):
    rng = random.Random(1)
    for i in range(runs):
        L = rng.choice([1, 2, 3, 5, 20])
        md = rng.choice([1, 2, 4, 8, 512])
        dil, d = [], 1
        for _ in range(L):
            dil.append(d); d = d * 2 if d * 2 <= md else 1
        kw = dict(L=L, S=rng.choice([128, 256]), NC=rng.choice([1, 2]), steps=rng.choice([2, 3, 4]), dil=dil, dump_last=rng.random() < 0.4,
                  t0=rng.choice([0, 0, 1, 7, 600]), slow=rng.choice([None, {"B": 4.0}, {"A": 3.0}, {"C": 5.0}, {"E": 3.0}, {"P": 6.0}, {"B": 0.3, "E": 0.3}]))
        try:
            trial(i, **kw)
        except Hazard as h:
            print("HAZARD in trial", i, kw, "\n  ", h)
            return 1
    print(f"{runs} randomised trials: no deadlock, no phase aliasing, no late commit, ring order consistent, no tile overwritten while read")
    return 0


if __name__ == "__main__":
    sys.exit(main(int(sys.argv[1]) if len(sys.argv) > 1 else 200))
