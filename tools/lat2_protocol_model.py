"""Discrete-event model of the synchronisation protocol of the three-CTA cluster kernel (csrc/wn_lat_kernel.cu, wn_lat2_kernel):
chain / tail / prep CTAs, each with eight compute warps and a weight-ring producer lane (and the chain CTA's sync warp, which waits
on its mbarriers for the compute warps and joins their named barrier), exchange mbarrier phases, transaction
bytes (st.async ... complete_tx), ring slots and tile buffers in the order the kernel does, with randomised latencies.  It checks
what a passing GPU run cannot show:

  * deadlock: every warp must finish every sample;
  * phase aliasing: a parity wait passes iff (completions - awaited) is odd -- a waiter two completions behind blocks for ever,
    three behind passes early; the model flags any wait that is ever two or more behind;
  * buffer hazards: a ring slot, an h tile, a pre-activation tile, a staged history / conditioning slot, the output layers' OB0 /
    OB1 tiles and the logits buffer must not be rewritten before every warp that reads its previous occupant has read it, and
    every reader must find the occupant it expects;
  * history visibility: the prep CTA stages x_l[t-d] from global memory with plain loads -- the chain CTA must have finished the step
    that wrote it; the model reports the smallest distance (in chain steps) it saw, which is what `L >= 12` in wn_launch_lat buys.

The chain CTA's weight ring has `nslot0` slots (2 or 3; the kernel's CfgC::NSLOT0).  With `wcur_ahead` (CfgC::WCUR_AHEAD) the
compute warps read the Wcur fragments of step n + 1 behind the h barrier of step n, and the sync warp waits for ring piece n + 1
before that barrier; without it they read them behind the x barrier of step n, and the sync warp waits for piece n before the
x barrier.  By default both follow the kernel: read ahead with three slots for 8 rows, behind the x barrier with two for 16.

Byte counts are those of a cluster of `rows` utterances (16, or 8 when all 8-row clusters are resident): every flow moves
rows / 16 of its 16-row bytes, with the same arrival counts.

Pure Python, no GPU.  `python tools/lat2_protocol_model.py [runs]` runs random trials; tests/test_lat2_protocol_model.py runs a
bounded number plus mutations (each re-introduces a defect and the model must see it).  Keep in step with the kernel source.
"""
import heapq
import random
import sys

NCW = 8          # compute warps per CTA
NAP = 4          # pre-activation tile buffers (chain CTA)
TSLOTS = 3       # tail ring slots (Wskip_l)
NPS = 8          # staged history / conditioning slots (prep CTA)
STAGE_AHEAD = 3  # the prep CTA stages tile n + 3 while it works on tile n


class Hazard(Exception):
    pass


class Barrier:
    """mbarrier with an arrival count and a transaction-byte count; completion k is the (k+1)-th phase flip."""

    def __init__(self, sim, name, count):
        self.sim, self.name, self.count = sim, name, count
        self.pending, self.tx, self.completed = count, 0, 0
        self.waiters = []                                   # (proc, awaited completion)

    def _check(self):
        if self.pending == 0 and self.tx == 0:
            self.completed += 1
            self.pending = self.count
            still = []
            for proc, k in self.waiters:
                behind = self.completed - k
                if behind >= 2:
                    raise Hazard(f"{proc.name}: {self.name} completed {self.completed} times while it waits for completion #{k} (phase aliasing)")
                if behind == 1:
                    self.sim.wake(proc, self.sim.lat(40, 120))
                else:
                    still.append((proc, k))
            self.waiters = still

    def arrive(self):
        if self.pending == 0:
            raise Hazard(f"{self.name}: more arrivals than its count in one phase")
        self.pending -= 1
        self._check()

    def expect_tx(self, nbytes):                            # mbarrier.arrive.expect_tx
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._check()


class Proc:
    def __init__(self, name, gen):
        self.name, self.gen, self.done = name, gen, False


class Sim:
    def __init__(self, L=12, T=3, seed=0, slow=None, bug=None, max_dil=4, rows=16, nslot0=None, wcur_ahead=None):
        wcur_ahead = rows == 8 if wcur_ahead is None else wcur_ahead
        nslot0 = nslot0 or (3 if wcur_ahead else 2)
        assert rows in (8, 16) and nslot0 in (2, 3)
        self.L, self.T, self.rows = L, T, rows
        self.nslot0, self.wcur_ahead = nslot0, wcur_ahead
        self.rng = random.Random(seed)
        self.slow = slow or {}
        self.bug = bug
        self.now, self.q, self.seq = 0, [], 0
        self.procs = []
        d, self.dil = 1, []
        for _ in range(L):
            self.dil.append(d)
            d = d * 2 if d * 2 <= max_dil else 1
        B = lambda n, c: Barrier(self, n, c)
        # chain CTA
        self.c_full = [B(f"chain.full{i}", 1) for i in range(nslot0)]
        self.c_empty = [B(f"chain.empty{i}", 1) for i in range(nslot0)]      # arrived by the sync warp
        self.hfree = [B(f"chain.hfree{i}", NCW) for i in range(2)]
        self.yfull = B("chain.yfull", 1)
        self.apfull = [B(f"chain.apfull{i}", 1) for i in range(NAP)]
        # tail CTA
        self.t_full = [B(f"tail.full{i}", 1) for i in range(TSLOTS)]
        self.t_empty = [B(f"tail.empty{i}", NCW) for i in range(TSLOTS)]
        self.hfull = [B(f"tail.hfull{i}", 1) for i in range(2)]
        # output layers (tail = columns 0-127, prep = 128-255): relu(skip) tail -> prep, relu(Zs) halves both ways, logits prep -> tail
        self.ob0full = B("prep.ob0full", 1)
        self.ob0free = B("tail.ob0free", NCW)
        self.ob1full = {c: B(f"{c}.ob1full", 1) for c in ("tail", "prep")}
        self.ob1free = {c: B(f"{c}.ob1free", 2 * NCW) for c in ("tail", "prep")}   # arrived by the warps of both CTAs
        self.lfull = B("tail.lfull", 1)
        self.lfree = B("prep.lfree", NCW)
        # prep CTA
        self.p_full = [B(f"prep.full{i}", 1) for i in range(4)]
        self.p_empty = [B(f"prep.empty{i}", NCW) for i in range(4)]
        self.pfull = [B(f"prep.pfull{i}", 4) for i in range(NPS)]          # warps 0-3 stage the history tile (128 thread arrivals)
        self.apfree = [B(f"prep.apfree{i}", 1) for i in range(NAP)]          # arrived by the chain's sync warp
        # armed by their owners one phase ahead (kernel prologue)
        self.yfull.expect_tx(self.nb(128))
        for b in self.apfull:
            b.expect_tx(self.nb(8192))
        for b in self.hfull:
            b.expect_tx(self.nb(2048))
        self.ob0full.expect_tx(self.nb(8192))
        for b in self.ob1full.values():
            b.expect_tx(self.nb(4096))
        self.lfull.expect_tx(self.nb(8192))
        # buffers: occupant tag + how many warps have read it
        self.slot = {}                                       # name -> [tag, reads]
        self.chain_steps_done = 0                            # steps whose x output (history ring write) is complete, all warps
        self.chain_step_warps = {}                           # step -> warps that finished it
        self.emb_done = {}                                   # sample -> warps that wrote the embedding
        self.min_history_margin = None
        self.nsteps = T * L

    def nb(self, bytes16):                                   # bytes of a flow that moves `bytes16` for 16 rows
        return bytes16 * self.rows // 16

    # ------------------------------------------------------------------ engine
    def lat(self, lo, hi, who=None):
        m = self.slow.get(who, 1.0) if who else 1.0
        return int(self.rng.randint(lo, hi) * m)

    def wake(self, proc, delay):
        self.seq += 1
        heapq.heappush(self.q, (self.now + delay, self.seq, proc))

    def spawn(self, name, gen):
        p = Proc(name, gen)
        self.procs.append(p)
        self.wake(p, 0)
        return p

    def after(self, delay, fn):                              # deferred side effect (a copy or a remote store landing)
        self.spawn(f"event@{self.now + delay}", self._delayed(delay, fn))

    def _delayed(self, delay, fn):
        yield ("delay", delay)
        fn()

    def run(self, limit=50_000_000):
        while self.q:
            self.now, _, proc = heapq.heappop(self.q)
            if self.now > limit:
                raise Hazard("time limit")
            try:
                while True:
                    op = next(proc.gen)
                    if op[0] == "delay":
                        self.wake(proc, op[1])
                        break
                    if op[0] == "wait":
                        bar, k = op[1], op[2]
                        behind = bar.completed - k
                        if behind >= 2:
                            raise Hazard(f"{proc.name}: starts waiting for completion #{k} of {bar.name}, which has completed {bar.completed} times (phase aliasing)")
                        if behind == 1:
                            continue
                        bar.waiters.append((proc, k))
                        break
            except StopIteration:
                proc.done = True
        stuck = [p.name for p in self.procs if not p.done]
        if stuck:
            raise Hazard("deadlock: " + ", ".join(sorted(stuck)[:12]))

    # ------------------------------------------------------------------ buffers
    def write(self, name, tag, readers):
        old = self.slot.get(name)
        if old is not None and old[1] < old[2]:
            raise Hazard(f"{name}: occupant {old[0]} overwritten by {tag} after {old[1]} of {old[2]} reads")
        self.slot[name] = [tag, 0, readers]

    def touch(self, name, tag, readers):                     # several senders fill one buffer: the first bytes to land claim it
        cur = self.slot.get(name)
        if cur is None or cur[0] != tag:
            self.write(name, tag, readers)

    def read(self, who, name, tag):
        cur = self.slot.get(name)
        if cur is None or cur[0] != tag:
            raise Hazard(f"{who}: expects {tag} in {name}, finds {cur[0] if cur else None}")
        cur[1] += 1

    # ------------------------------------------------------------------ roles
    def producer(self, who, full, empty, nslots, pieces, slotname, readers=NCW):
        for n, nbytes in enumerate(pieces):
            sl = n % nslots
            yield ("wait", empty[sl], n // nslots - 1)
            full[sl].expect_tx(nbytes)

            def land(n=n, sl=sl, nbytes=nbytes):
                self.write(f"{slotname}{sl}", n, readers)
                full[sl].complete_tx(nbytes)
            self.after(self.lat(300, 900, who), land)
            yield ("delay", self.lat(20, 60, who))

    def chain_warp(self, w):
        """A compute warp of the chain CTA: its layer step waits only on the CTA barrier it shares with the sync warp."""
        who = f"chain.w{w}"
        L, T, ns = self.L, self.T, self.nslot0
        yield from self.cta_bar("chain", who)
        if self.nsteps:
            self.read(who, "ap0", 0)                         # pre-activation tile 0 (the sync warp saw it land)
            if self.wcur_ahead:
                self.read(who, "cring0", 0)                  # Wcur of step 0 (so did ring piece 0)
        k = 0
        for t in range(T):
            if t > 0:
                yield ("wait", self.yfull, t - 1)
                if w == 0 and t + 1 < T:
                    self.yfull.expect_tx(self.nb(128))
            yield ("delay", self.lat(150, 300, who))         # embedding, history write of (t, layer 0)
            self.emb_done[t] = self.emb_done.get(t, 0) + 1
            yield from self.cta_bar("chain", who)            # x barrier
            for l in range(L):
                if not self.wcur_ahead:
                    self.read(who, f"cring{k % ns}", k)      # Wcur of this step
                yield ("delay", self.lat(100, 200, who))     # cur GEMM
                self.read(who, f"cring{k % ns}", k)          # Wres of this step, under the gate
                yield ("delay", self.lat(100, 200, who))     # gate

                def land_h(k=k):                             # this warp's 256 (8 rows: 128) bytes of the h tile + their complete_tx
                    self.touch(f"h{k & 1}", k, NCW)          # (the tail's buffer is free: the sync warp waited before the x barrier)
                    self.hfull[k & 1].complete_tx(self.nb(256))
                self.after(self.lat(200, 700), land_h)
                yield from self.cta_bar("chain", who)        # h barrier
                if k + 1 < self.nsteps:
                    self.read(who, f"ap{(k + 1) % NAP}", k + 1)
                yield ("delay", self.lat(150, 300, who))     # res GEMM (weights of the same piece)
                if self.wcur_ahead and k + 1 < self.nsteps:
                    self.read(who, f"cring{(k + 1) % ns}", k + 1)   # Wcur of the next step (the sync warp saw its piece land)
                yield ("delay", self.lat(30, 80, who))       # x tile + history ring write of (t, l + 1)
                self.chain_step_warps[k] = self.chain_step_warps.get(k, 0) + 1
                while self.chain_step_warps.get(self.chain_steps_done, 0) == NCW:
                    self.chain_steps_done += 1
                if l + 1 < L:
                    yield from self.cta_bar("chain", who)    # x barrier
                k += 1

    def chain_sync(self):
        """The chain CTA's sync warp (lane 0): every mbarrier wait and hand-back of the layer loop."""
        who = "chain.sync"
        ns, ahead = self.nslot0, self.wcur_ahead
        if self.nsteps:
            yield ("wait", self.apfull[0], 0)
            if ahead and self.bug != "no_full_wait":
                yield ("wait", self.c_full[0], 0)
        yield from self.cta_bar("chain", who)
        for n in range(self.nsteps):
            b, hb = n % NAP, n & 1
            if not ahead and self.bug != "no_full_wait":
                yield ("wait", self.c_full[n % ns], n // ns)
            if self.bug not in ("no_hfree", "hfree_late"):   # the tail has read h tile n - 2: the compute warps may send tile n
                yield ("wait", self.hfree[hb], (n >> 1) - 1)
            yield from self.cta_bar("chain", who)            # x barrier of step n: pre-activation tile n has been read
            if self.bug == "hfree_late":
                yield ("wait", self.hfree[hb], (n >> 1) - 1)
            self.apfull[b].expect_tx(self.nb(8192))          # armed for the tile NAP steps on, before the "free" signal
            if self.bug != "no_apfree":
                self.after(self.lat(150, 400), self.apfree[b].arrive)
            if self.bug == "empty_early":                    # (Wres of piece n is still to be read)
                self.c_empty[n % ns].arrive()
            if n + 1 < self.nsteps and self.bug != "no_apfull_wait":
                yield ("wait", self.apfull[(n + 1) % NAP], (n + 1) // NAP)
            if ahead and n + 1 < self.nsteps and self.bug not in ("no_full_wait", "no_early_full_wait"):
                yield ("wait", self.c_full[(n + 1) % ns], (n + 1) // ns)
            yield from self.cta_bar("chain", who)            # h barrier of step n: ring piece n has been read
            if self.bug not in ("no_empty", "empty_early"):
                self.c_empty[n % ns].arrive()
            yield ("delay", self.lat(10, 40, who))

    def cta_bar(self, cta, who):                             # bar.sync among the compute warps of one CTA (+ the chain's sync warp)
        bar = self.__dict__.setdefault("_barobj", {}).setdefault(cta, Barrier(self, f"{cta}.bar.sync", NCW + (cta == "chain")))
        mine = bar.completed
        bar.arrive()
        if bar.completed == mine:
            yield ("wait", bar, mine)
        else:
            yield ("delay", self.lat(30, 60))

    def tail_warp(self, w):
        who = f"tail.w{w}"
        L, T = self.L, self.T
        pc = hc = 0
        for t in range(T):
            for l in range(L):
                yield ("wait", self.hfull[hc & 1], hc >> 1)
                self.read(who, f"h{hc & 1}", hc)
                yield ("wait", self.t_full[pc % TSLOTS], pc // TSLOTS)
                self.read(who, f"tring{pc % TSLOTS}", pc)
                yield ("delay", self.lat(250, 500, who))     # skip GEMM
                if w == 0:
                    self.hfull[hc & 1].expect_tx(self.nb(2048))   # armed for the tile after next, before this warp's "free" signal
                self.after(self.lat(150, 400), self.hfree[hc & 1].arrive)
                self.t_empty[pc % TSLOTS].arrive()
                pc += 1
                hc += 1
            # relu(skip + Bskip): this warp's 1 KB (8 rows: 512 B) into the prep CTA's OB0 (and its own, ordered by the CTA barrier)
            yield ("wait", self.ob0free, t - 1)

            def land_ob0(t=t):
                self.touch("prep.ob0", t, NCW)
                self.ob0full.complete_tx(self.nb(1024))
            self.after(self.lat(200, 700), land_ob0)
            yield from self.cta_bar("tail", who)
            yield from self.out_half("tail", w, t)
            self.touch("tail.lbuf", t, NCW)                  # this warp's logits of columns 0-127
            yield from self.cta_bar("tail", who)
            yield ("wait", self.lfull, t)                    # columns 128-255 from the prep CTA
            self.read(who, "tail.lbuf", t)
            yield ("delay", self.lat(800, 1500, who))        # softmax + sampling of this warp's two utterances (8 rows: one)
            if w == 0:
                self.lfull.expect_tx(self.nb(8192))                   # armed for the next sample, before this warp's "free" signal
            self.after(self.lat(150, 400), self.lfree.arrive)
            if t + 1 < T:
                self.after(self.lat(200, 700), lambda: self.yfull.complete_tx(self.nb(16)))
            yield from self.cta_bar("tail", who)

    def out_half(self, cta, w, t):
        """Zs -> relu(Zs) exchange -> Za of one CTA's 128 output columns (wn_lat2_kernel's out_half)."""
        who, peer = f"{cta}.w{w}", "prep" if cta == "tail" else "tail"
        if cta == "prep":
            yield ("wait", self.ob0full, t)
            self.read(who, "prep.ob0", t)
        yield ("delay", self.lat(300, 700, who))             # Zs GEMM, weights resident
        if cta == "prep":
            if w == 0:
                self.ob0full.expect_tx(self.nb(8192))
            self.after(self.lat(150, 400), self.ob0free.arrive)
        yield ("wait", self.ob1free[cta], t - 1)
        self.touch(f"{cta}.ob1", t, NCW)                     # this warp's 16 B (8 rows: 8 B) per thread, locally ...

        def land_ob1(t=t):                                   # ... and into the peer's OB1
            self.touch(f"{peer}.ob1", t, NCW)
            self.ob1full[peer].complete_tx(self.nb(512))
        self.after(self.lat(200, 700), land_ob1)
        yield from self.cta_bar(cta, who)
        if self.bug != "no_ob1full_wait":
            yield ("wait", self.ob1full[cta], t)
        self.read(who, f"{cta}.ob1", t)
        yield ("delay", self.lat(300, 900, who))             # Za GEMM
        if w == 0:
            self.ob1full[cta].expect_tx(self.nb(4096))
        self.ob1free[cta].arrive()
        self.after(self.lat(150, 400), self.ob1free[peer].arrive)

    def out_prep(self, w, t):
        yield from self.out_half("prep", w, t)
        yield ("wait", self.lfree, t - 1)

        def land_l(t=t):                                     # this warp's 1 KB (8 rows: 512 B) of logits into the tail CTA's buffer
            self.touch("tail.lbuf", t, NCW)
            self.lfull.complete_tx(self.nb(1024))
        self.after(self.lat(200, 700), land_l)

    def prep_warp(self, w):
        who = f"prep.w{w}"
        L = self.L
        pcnt = 0
        tout = 0                                             # the next sample whose output half is due

        def stage():
            nonlocal pcnt
            slot = pcnt % NPS
            if pcnt < self.nsteps:
                t, l = divmod(pcnt, L)
                # conditioning: this warp's own 512 (8 rows: 256) bytes; history: warps 0-3 copy the tile and arrive on pfull
                self.write(f"cond{slot}.w{w}", pcnt, 1)
                if w < 4:
                    d = self.dil[l]
                    if t - d >= 0:                           # (before the utterance: zeros; before t_begin: a previous launch)
                        src_step = (t - d) * L + l - 1       # chain step that wrote x_l[t-d] (layer 0: the embedding of that sample)
                        if l == 0:
                            if self.emb_done.get(t - d, 0) < NCW:
                                raise Hazard(f"{who}: stages x_0[{t - d}] before the chain CTA has written that embedding")
                            margin = self.chain_steps_done - (t - d) * L
                        else:
                            if self.chain_steps_done <= src_step:
                                raise Hazard(f"{who}: stages the history tile of step {pcnt} before the chain CTA finished step {src_step} (it has finished {self.chain_steps_done})")
                            margin = self.chain_steps_done - 1 - src_step
                        if self.min_history_margin is None or margin < self.min_history_margin:
                            self.min_history_margin = margin
                    self.touch(f"pst{slot}", pcnt, NCW)
                    self.after(self.lat(300, 900), self.pfull[slot].arrive)
            elif w < 4:
                self.pfull[slot].arrive()                    # (past the end: zero fill, immediate arrive)
            pcnt += 1

        for _ in range(STAGE_AHEAD):
            stage()
        for n in range(self.nsteps):
            b, slot = n % NAP, n % NPS
            self.read(who, f"cond{slot}.w{w}", n)
            yield ("wait", self.p_full[n & 3], n >> 2)
            self.read(who, f"pring{n & 3}", n)
            yield ("wait", self.pfull[slot], n // NPS)
            self.read(who, f"pst{slot}", n)
            yield ("delay", self.lat(200, 400, who))         # Wprev . x[t-d] + (Bh + Lh)
            self.p_empty[n & 3].arrive()
            if self.bug != "no_apfree_wait":
                yield ("wait", self.apfree[b], n // NAP - 1)

            def land_ap(n=n, b=b):                           # this warp's 1 KB (8 rows: 512 B) of the pre-activation tile + their complete_tx
                self.touch(f"ap{b}", n, NCW)
                self.apfull[b].complete_tx(self.nb(1024))
            self.after(self.lat(300, 900), land_ap)
            yield ("delay", self.lat(100, 400, who))         # the remote stores occupy this CTA's load/store pipe
            stage()
            # the output half of sample tout: after step (tout + 1, 1) has been shipped, before the wait for the buffer of step
            # (tout + 1, NAP + 1) -- the chain CTA frees it only inside sample tout + 1 ("prep_out_late" waits past it: deadlock)
            due = (tout + 1) * L + 1 + (NAP if self.bug == "prep_out_late" else 0)
            if n == due:
                yield from self.out_prep(w, tout)
                tout += 1
        while tout < self.T:                                 # the last sample: no steps follow it
            yield from self.out_prep(w, tout)
            tout += 1

    def build(self):
        L, T = self.L, self.T
        self.spawn("chain.producer", self.producer("chain.producer", self.c_full, self.c_empty, self.nslot0, [24576] * (T * L), "cring", 2 * NCW))
        self.spawn("tail.producer", self.producer("tail.producer", self.t_full, self.t_empty, TSLOTS, [32768] * (T * L), "tring"))
        self.spawn("prep.producer", self.producer("prep.producer", self.p_full, self.p_empty, 4, [16384] * (T * L), "pring"))
        self.spawn("chain.sync", self.chain_sync())
        for w in range(NCW):
            self.spawn(f"chain.w{w}", self.chain_warp(w))
            self.spawn(f"tail.w{w}", self.tail_warp(w))
            self.spawn(f"prep.w{w}", self.prep_warp(w))
        return self


def trial(seed, **kw):
    rng = random.Random(seed)
    L = kw.pop("L", rng.choice([12, 13, 16, 20]))
    T = kw.pop("T", rng.choice([2, 3, 4]))
    slow = kw.pop("slow", None)
    rows = kw.pop("rows", 8 if seed % 2 == 0 else 16)        # (no draw from rng: the latencies of a seed do not depend on it)
    if slow is None and rng.random() < 0.6:
        slow = {rng.choice(["chain.w0", "chain.w5", "tail.w3", "prep.w1", "prep.w6", "chain.producer", "tail.producer", "prep.producer"]): rng.choice([0.3, 3.0, 10.0])}
    sim = Sim(L=L, T=T, seed=seed, slow=slow, max_dil=kw.pop("max_dil", rng.choice([1, 4, 512])), rows=rows, **kw).build()
    sim.run()
    return sim


if __name__ == "__main__":
    runs = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    worst = None
    for s in range(runs):
        sim = trial(s)
        if sim.min_history_margin is not None and (worst is None or sim.min_history_margin < worst):
            worst = sim.min_history_margin
    print(f"{runs} trials: no deadlock, no aliasing, no buffer hazard; smallest history margin seen: {worst} chain steps")
