"""Executable models of warp-specialised GEMM mbarrier protocols: the warp roles are coroutines, the barriers follow the PTX
semantics (arrival count, expect_tx / complete_tx byte credit, phase parity), asynchronous agents (TMA, the tensor core's in-order
completion queues) act after random delays, and a random scheduler interleaves everything.  Checked over many schedules and
shapes: no deadlock, a waiter is never lapped by its barrier (parity ambiguity), no shared-memory stage is overwritten before the
MMAs that read it have completed, every tile is produced exactly once.

``WgmmaModel`` is the protocol of csrc/gemm_wgmma.cu: one TMA producer, two consumer warpgroups that each issue a wgmma group per
stage, keep one group in flight (``wgmma.wait_group 1``) and only then release the PREVIOUS stage, ``empty`` armed with one
arrival per consumer warpgroup.  ``Model`` is a design this code base no longer ships (a dedicated MMA issuer whose commits
release stages, double-buffered tensor-memory accumulators, 1-CTA and 2-CTA forms); it is kept as a check of the barrier
arithmetic shared by both."""
import random

import pytest

A_BYTES, B_BYTES = 16384, 32768


class Barrier:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count
        assert self.pending >= 0, "more arrivals than the barrier was initialised for"

    def arrive(self):
        self.pending -= 1
        self._maybe_complete()

    def expect_tx(self, nbytes):  # mbarrier.arrive.expect_tx
        self.tx += nbytes
        self.pending -= 1
        self._maybe_complete()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._maybe_complete()


class Wait:
    """``mbarrier.try_wait.parity``: passes once the phase with this parity has completed.  ``k`` is the absolute phase index the
    kernel's arithmetic means; being lapped (barrier two phases ahead) would make the parity test lie."""

    def __init__(self, bar, k):
        self.bar, self.k = bar, k

    def ready(self):
        assert self.bar.phase <= self.k + 1, "waiter lapped by its barrier: parity is ambiguous"
        return self.bar.phase > self.k


def wait_parity(bar, parity, k):
    # what the kernel computes is only `parity`; k is the phase index that parity is supposed to denote
    assert parity == (k & 1), "kernel parity arithmetic disagrees with the intended phase"
    return Wait(bar, k)


class Model:
    def __init__(self, ctas, stages, tiles, num_kb, seed):
        self.rng = random.Random(seed)
        self.ctas, self.S, self.tiles, self.num_kb = ctas, stages, tiles, num_kb
        n_epi = 4 * ctas
        self.full = [Barrier(ctas) for _ in range(stages)]                               # leader's
        self.empty = [[Barrier(1) for _ in range(stages)] for _ in range(ctas)]          # one set per CTA (multicast commit)
        self.acc_full = [[Barrier(1) for _ in range(2)] for _ in range(ctas)]
        self.acc_empty = [Barrier(n_epi) for _ in range(2)]                              # leader's
        self.smem = [[None] * stages for _ in range(ctas)]       # (tile, kb) resident in stage s of CTA c, None = free
        self.inflight_reads = [[0] * stages for _ in range(ctas)]
        self.tmem = [None, None]                                  # tile whose result is complete in accumulator a
        self.tmem_readers = [0, 0]                                # epilogue warps still to read accumulator a
        self.async_q = []                                         # [delay, fn] agents (TMA engines)
        self.mma_q = []                                           # in-order tensor-core completion queue: fn
        self.done_tiles = []

    # ---- asynchronous agents -------------------------------------------------------------------------------------
    def later(self, fn):
        self.async_q.append([self.rng.randint(0, 6), fn])

    def step_agents(self):
        progressed = False
        for item in list(self.async_q):
            if item[0] <= 0:
                self.async_q.remove(item)
                item[1]()
                progressed = True
            else:
                item[0] -= 1
                progressed = True
        if self.mma_q and self.rng.random() < 0.6:
            self.mma_q.pop(0)()
            progressed = True
        return progressed

    # ---- warp roles ----------------------------------------------------------------------------------------------
    def producer(self, c):
        it = 0
        for tile in range(self.tiles):
            for kb in range(self.num_kb):
                s = it % self.S
                k = it // self.S
                yield wait_parity(self.empty[c][s], ((it // self.S) & 1) ^ 1, k - 1)   # k-th use waits for the (k-1)-th release
                if c == 0:
                    self.full[s].expect_tx(self.ctas * (A_BYTES + B_BYTES // self.ctas))
                else:
                    self.full[s].arrive()

                def land(c=c, s=s, tile=tile, kb=kb, nbytes=A_BYTES + B_BYTES // self.ctas):
                    assert self.smem[c][s] is None and self.inflight_reads[c][s] == 0, "TMA overwrote a stage that is still being read"
                    self.smem[c][s] = (tile, kb)
                    self.full[s].complete_tx(nbytes)

                self.later(land)
                it += 1
                yield None

    def mma(self):
        it = 0
        for local, tile in enumerate(range(self.tiles)):
            acc = local & 1
            yield wait_parity(self.acc_empty[acc], ((local >> 1) & 1) ^ 1, (local >> 1) - 1)
            assert self.tmem_readers[acc] == 0, "MMA overwrites an accumulator that an epilogue warp still reads"
            self.tmem[acc] = None
            for kb in range(self.num_kb):
                s = it % self.S
                yield wait_parity(self.full[s], (it // self.S) & 1, it // self.S)
                for c in range(self.ctas):
                    assert self.smem[c][s] == (tile, kb), f"stage {s} of CTA {c} holds {self.smem[c][s]}, MMA expects {(tile, kb)}"
                    self.inflight_reads[c][s] += 1

                def mma_done(s=s):
                    for c in range(self.ctas):
                        self.inflight_reads[c][s] -= 1
                        self.smem[c][s] = None

                def commit_empty(s=s):  # tcgen05.commit → (multicast) arrive on empty[s] of every CTA of the group
                    for c in range(self.ctas):
                        self.empty[c][s].arrive()

                self.mma_q += [mma_done, commit_empty]
                it += 1
                yield None

            def commit_acc(acc=acc, tile=tile):
                self.tmem[acc] = tile
                self.tmem_readers[acc] = 4 * self.ctas
                for c in range(self.ctas):
                    self.acc_full[c][acc].arrive()

            self.mma_q.append(commit_acc)
            yield None

    def epilogue(self, c, w):
        for local, tile in enumerate(range(self.tiles)):
            acc = local & 1
            yield wait_parity(self.acc_full[c][acc], (local >> 1) & 1, local >> 1)
            assert self.tmem[acc] == tile, f"epilogue of tile {tile} reads accumulator holding {self.tmem[acc]}"
            for _ in range(self.rng.randint(0, 3)):
                yield None  # tcgen05.ld + stores take a while
            assert self.tmem[acc] == tile
            self.tmem_readers[acc] -= 1
            if c == 0 and w == 0:
                self.done_tiles.append(tile)
            self.acc_empty[acc].arrive()   # CTA 1 arrives remotely (mapa + mbarrier.arrive.shared::cluster)
            yield None

    def run(self):
        actors = [self.producer(c) for c in range(self.ctas)] + [self.mma()] + [self.epilogue(c, w) for c in range(self.ctas) for w in range(4)]
        blocked = {id(a): None for a in actors}
        live = list(actors)
        idle_rounds = 0
        while live:
            progressed = self.step_agents()
            self.rng.shuffle(live)
            for a in list(live):
                w = blocked[id(a)]
                if w is not None and not w.ready():
                    continue
                try:
                    blocked[id(a)] = next(a)
                    progressed = True
                except StopIteration:
                    live.remove(a)
                    progressed = True
            idle_rounds = 0 if (progressed or self.async_q or self.mma_q) else idle_rounds + 1
            assert idle_rounds < 3, "deadlock: every warp role is blocked and no asynchronous work is pending"
        while self.async_q or self.mma_q:
            self.step_agents()
        assert self.done_tiles == list(range(self.tiles))
        assert all(x is None for row in self.smem for x in row)


@pytest.mark.parametrize("ctas,stages", [(1, 4), (1, 6), (2, 6)])
def test_gemm_pipeline_protocol_has_no_deadlock_or_hazard(ctas, stages):
    rng = random.Random(ctas * 100 + stages)
    for seed in range(150):
        tiles, num_kb = rng.randint(1, 7), rng.choice([1, 2, 3, stages - 1, stages, stages + 1, 16])
        Model(ctas, stages, tiles, num_kb, seed).run()


def test_model_detects_a_wrong_arrival_count():
    """The model is only worth something if it fails for a broken protocol: with ``acc_empty`` initialised for 4 arrivals in the
    2-CTA kernel (the 1-CTA value) the leader would reuse an accumulator while the peer's epilogue still reads it."""
    failures = 0
    for seed in range(40):
        m = Model(2, 6, 5, 3, seed)
        m.acc_empty = [Barrier(4) for _ in range(2)]
        try:
            m.run()
        except AssertionError:
            failures += 1
    assert failures > 0


class Until:
    def __init__(self, cond):
        self.cond = cond

    def ready(self):
        return self.cond()


class WgmmaModel:
    """csrc/gemm_wgmma.cu: full[s] (1 arrival + expect_tx), empty[s] (``empty_count`` arrivals, 2 in the kernel)."""

    def __init__(self, stages, tiles, num_kb, seed, empty_count=2):
        self.rng = random.Random(seed)
        self.S, self.tiles, self.num_kb = stages, tiles, num_kb
        self.full = [Barrier(1) for _ in range(stages)]
        self.empty = [Barrier(empty_count) for _ in range(stages)]
        self.smem = [None] * stages          # (tile, kb) resident in stage s
        self.reads = [0] * stages            # wgmma groups still reading stage s
        self.groups = [[], []]               # per consumer warpgroup: stages of its outstanding groups, completed in order
        self.async_q = []
        self.done = [[], []]

    def step_agents(self):
        progressed = False
        for item in list(self.async_q):
            progressed = True
            if item[0] <= 0:
                self.async_q.remove(item)
                item[1]()
            else:
                item[0] -= 1
        for q in self.groups:
            if q and self.rng.random() < 0.5:
                self.reads[q.pop(0)] -= 1
                progressed = True
        return progressed

    def producer(self):
        it = 0
        for tile in range(self.tiles):
            for kb in range(self.num_kb):
                s, k = it % self.S, it // self.S
                yield wait_parity(self.empty[s], (k & 1) ^ 1, k - 1)
                self.full[s].expect_tx(A_BYTES + B_BYTES)

                def land(s=s, tile=tile, kb=kb):
                    assert self.reads[s] == 0, "TMA overwrote a stage that a wgmma group still reads"
                    self.smem[s] = (tile, kb)
                    self.full[s].complete_tx(A_BYTES + B_BYTES)

                self.async_q.append([self.rng.randint(0, 6), land])
                it += 1
                yield None

    def consumer(self, cw):
        it = 0
        for tile in range(self.tiles):
            prev = None
            for kb in range(self.num_kb):
                s = it % self.S
                yield wait_parity(self.full[s], (it // self.S) & 1, it // self.S)
                assert self.smem[s] == (tile, kb), f"consumer {cw} expects {(tile, kb)} in stage {s}, finds {self.smem[s]}"
                self.reads[s] += 1
                self.groups[cw].append(s)                                   # wgmma x4 + commit_group
                yield Until(lambda cw=cw: len(self.groups[cw]) <= 1)        # wait_group 1: the previous group is done
                if prev is not None:
                    self.empty[prev].arrive()
                prev = s
                it += 1
            yield Until(lambda cw=cw: not self.groups[cw])                 # wait_group 0
            self.empty[prev].arrive()
            for _ in range(self.rng.randint(0, 3)):
                yield None                                                  # epilogue from registers
            self.done[cw].append(tile)

    def run(self):
        actors = [self.producer(), self.consumer(0), self.consumer(1)]
        blocked = {id(a): None for a in actors}
        live, idle_rounds = list(actors), 0
        while live:
            progressed = self.step_agents()
            self.rng.shuffle(live)
            for a in list(live):
                w = blocked[id(a)]
                if w is not None and not w.ready():
                    continue
                try:
                    blocked[id(a)] = next(a)
                except StopIteration:
                    live.remove(a)
                progressed = True
            idle_rounds = 0 if (progressed or self.async_q or any(self.groups)) else idle_rounds + 1
            assert idle_rounds < 3, "deadlock: every warp role is blocked and no asynchronous work is pending"
        assert self.done == [list(range(self.tiles))] * 2


@pytest.mark.parametrize("stages", [4, 6])
def test_wgmma_stage_ring_has_no_deadlock_or_hazard(stages):
    rng = random.Random(stages)
    for seed in range(200):
        tiles, num_kb = rng.randint(1, 7), rng.choice([1, 2, 3, stages - 1, stages, stages + 1, 16])
        WgmmaModel(stages, tiles, num_kb, seed).run()


def test_wgmma_model_detects_a_single_arrival_empty_barrier():
    """With ``empty`` armed for one arrival the first consumer to release a stage would let TMA overwrite it while the other
    consumer's wgmma group still reads it."""
    failures = 0
    for seed in range(60):
        try:
            WgmmaModel(4, 4, 6, seed, empty_count=1).run()
        except AssertionError:
            failures += 1
    assert failures > 0


# ---- symmetric-buffer reuse of the fused fc2+combine path (ops/moe_peer.py: linear_push_gather) ---------------------------------
class EpochBarrier:
    """peer_barrier(ctx, epoch) of csrc/peer.cuh: every rank publishes ``epoch`` to all peers and waits until all have."""

    def __init__(self, world):
        self.seen = [[0] * world for _ in range(world)]   # seen[r][p]: the epoch of rank p as visible on rank r

    def arrive(self, rank, epoch):
        for r in range(len(self.seen)):
            self.seen[r][rank] = epoch

    def passed(self, rank, epoch):
        return all(e >= epoch for e in self.seen[rank])


def _moe_rank(rank, world, layers, bar, buf, reading, rng):
    """Kernel sequence of one rank for ``layers`` MoE layers sharing ONE symmetric buffer: the GEMM epilogue pushes this rank's expert
    outputs into every peer's buffer (no entry barrier), then the local-layout gather kernel: barrier, read own buffer, barrier."""
    epoch = 0
    for layer in range(layers):
        for dst in rng.sample(range(world), world):            # PEER epilogue: tiles leave in any order
            assert reading[dst] == 0 or buf[dst][rank] == layer, f"layer {layer} overwrites rank {dst}'s buffer while it still reads layer {buf[dst][rank]}"
            buf[dst][rank] = layer
            yield None
        bar.arrive(rank, epoch + 1)                              # gather kernel, entry barrier: all pushes of this layer have landed
        while not bar.passed(rank, epoch + 1):
            yield None
        reading[rank] += 1
        for src in range(world):
            assert buf[rank][src] == layer, f"rank {rank} gathers layer {layer} but the slot of rank {src} holds layer {buf[rank][src]}"
            yield None
        reading[rank] -= 1
        bar.arrive(rank, epoch + 2)                              # exit barrier: nobody may recycle the buffers before every reader is done
        while not bar.passed(rank, epoch + 2):
            yield None
        epoch += 2


@pytest.mark.parametrize("world", [2, 4, 8])
def test_fused_combine_buffer_reuse_is_race_free(world):
    for seed in range(60):
        rng = random.Random(seed)
        bar, buf, reading = EpochBarrier(world), [[-1] * world for _ in range(world)], [0] * world
        ranks = [_moe_rank(r, world, 5, bar, buf, reading, rng) for r in range(world)]
        live = list(ranks)
        guard = 0
        while live:
            a = rng.choice(live)               # arbitrary relative speeds of the ranks
            try:
                next(a)
            except StopIteration:
                live.remove(a)
            guard += 1
            assert guard < 200000, "livelock"


def test_the_buffer_model_needs_the_exit_barrier():
    """Without the second barrier a fast rank's next push lands in a buffer that a slow rank is still gathering from."""
    def no_exit_barrier(rank, world, layers, bar, buf, reading, rng):
        epoch = 0
        for layer in range(layers):
            for dst in range(world):
                assert reading[dst] == 0 or buf[dst][rank] == layer
                buf[dst][rank] = layer
                yield None
            bar.arrive(rank, epoch + 1)
            while not bar.passed(rank, epoch + 1):
                yield None
            reading[rank] += 1
            for src in range(world):
                assert buf[rank][src] == layer
                yield None
            reading[rank] -= 1
            epoch += 1

    failures = 0
    for seed in range(40):
        rng = random.Random(seed)
        world = 4
        bar, buf, reading = EpochBarrier(world), [[-1] * world for _ in range(world)], [0] * world
        live = [no_exit_barrier(r, world, 4, bar, buf, reading, rng) for r in range(world)]
        try:
            while live:
                a = rng.choice(live)
                try:
                    next(a)
                except StopIteration:
                    live.remove(a)
        except AssertionError:
            failures += 1
    assert failures > 0
