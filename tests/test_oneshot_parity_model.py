"""Schedule-exploring model of the one-shot all-reduce's double-buffered staging area (bagua_b200/csrc/peer_kernels.cu,
``allreduce_oneshot_kernel``): every rank pushes its message into slot [parity][rank] of every peer, ONE per-CTA-row barrier, then
reduces the slots it received.  Calls use different grid sizes (1-8 CTAs by message size, ``PeerEngine.launch_cfg``).

The round-1 kernel took the parity from the per-CTA epoch; CTAs that sit out small calls then fall out of step with CTA 0 and a
fast rank can overwrite a slot a slow peer is still reading (ADVICE.md; the comment on ``parity`` in ``allreduce_oneshot_kernel``).  The fix takes the parity from a
per-communicator CALL counter kept by the host (``PeerComm::next_oneshot_parity``).  The model executes random interleavings of the
CTAs of 2-3 ranks over random call sequences, with per-rank stream order (kernel c+1 starts when kernel c has retired) and the
real barrier rule (row b waits for row b of every peer), and checks every read: each slot must hold exactly the data of THIS call.
The old parity rule must be caught by the same checker."""
import random

import pytest


def run_schedule(nranks, grids, nvec, rng, parity_from_call):
    ncalls = len(grids)
    staging = [[[[None] * nvec for _ in range(nranks)] for _ in range(2)] for _ in range(nranks)]   # [owner][parity][source][vector] = call id
    flags = [[[0] * nranks for _ in range(8)] for _ in range(nranks)]                               # [owner][row][source] = epoch
    epochs = [[0] * 8 for _ in range(nranks)]
    call_of = [0] * nranks            # kernel each rank is currently executing
    ctas = [None] * nranks            # per rank: list of CTA states of the running kernel

    def start(r):
        c = call_of[r]
        ctas[r] = [{"pc": "write", "row": b, "parity": (c & 1) if parity_from_call else (epochs[r][b] & 1), "epoch": epochs[r][b] + 1} for b in range(grids[c])]

    for r in range(nranks):
        start(r)
    steps = 0
    while any(call_of[r] < ncalls for r in range(nranks)):
        steps += 1
        assert steps < 100_000, "no progress (deadlock in the model)"
        runnable = []
        for r in range(nranks):
            if call_of[r] >= ncalls:
                continue
            for i, cta in enumerate(ctas[r]):
                if cta["pc"] == "wait" and not all(flags[r][cta["row"]][p] >= cta["epoch"] for p in range(nranks)):
                    continue
                if cta["pc"] != "done":
                    runnable.append((r, i))
        r, i = rng.choice(runnable)
        cta, c, g = ctas[r][i], call_of[r], grids[call_of[r]]
        mine = [v for v in range(nvec) if v % g == cta["row"]]
        if cta["pc"] == "write":
            for p in range(nranks):
                for v in mine:
                    staging[p][cta["parity"]][r][v] = c
            cta["pc"] = "arrive"
        elif cta["pc"] == "arrive":      # st.release.sys of the epoch into every peer's row
            for p in range(nranks):
                flags[p][cta["row"]][r] = cta["epoch"]
            cta["pc"] = "wait"
        elif cta["pc"] == "wait":
            cta["pc"] = "read"
        elif cta["pc"] == "read":
            for src in range(nranks):
                for v in mine:
                    got = staging[r][cta["parity"]][src][v]
                    if got != c:
                        return f"rank {r} call {c} (grid {g}) row {cta['row']}: slot of rank {src}, vector {v} holds call {got}"
            epochs[r][cta["row"]] = cta["epoch"]
            cta["pc"] = "done"
        if all(x["pc"] == "done" for x in ctas[r]):     # the kernel retires; the next one on the stream may start
            call_of[r] += 1
            if call_of[r] < ncalls:
                start(r)
    return None


def _sequences(seed, n):
    rng = random.Random(seed)
    for _ in range(n):
        yield [rng.choice([1, 1, 2, 3, 4]) for _ in range(rng.randint(3, 7))], rng.randint(2, 3), random.Random(rng.random())


def test_host_call_counter_parity_never_exposes_a_slot_under_mixed_grid_sizes():
    for grids, nranks, rng in _sequences(seed=7, n=400):
        for _ in range(5):
            assert run_schedule(nranks, grids, nvec=12, rng=rng, parity_from_call=True) is None, (grids, nranks)


def test_per_cta_epoch_parity_is_caught_by_the_model():
    """The round-1 rule: a small call advances only CTA 0's epoch, so in the next large call the rows disagree about the parity —
    rows > 0 reuse the half they used last, which a slower peer may still be reading, or read a half nobody wrote for this call."""
    found = None
    for grids, nranks, rng in _sequences(seed=7, n=400):
        for _ in range(5):
            found = found or run_schedule(nranks, grids, nvec=12, rng=rng, parity_from_call=False)
        if found:
            break
    assert found is not None, "the checker failed to find the known hazard"


@pytest.mark.parametrize("grids", [[1, 4, 1, 4, 4], [4, 1, 1, 4], [2, 3, 2, 3, 1, 4]])
def test_named_mixed_grid_sequences(grids):
    for seed in range(40):
        assert run_schedule(3, grids, nvec=12, rng=random.Random(seed), parity_from_call=True) is None


# ---------------------------------------------------------------------------------------------------------------------
# peer_barrier_vote (bagua_b200/csrc/peer.cuh): ONE vote area per communicator, no double buffering
# ---------------------------------------------------------------------------------------------------------------------
def run_vote_schedule(nranks, ncta, nlaunches, rng, closing_barrier):
    """Every launch: each CTA of rank r deposits the rank's word for this launch in slot [r] of every peer's vote area, releases its
    row flag, acquires the peers' flags, reads the P words of its own area — and (async_average_kernel) later passes the kernel's
    closing barrier.  Stream order per rank; per-row barriers.  A read must see every peer's word of THIS launch."""
    votes = [[None] * nranks for _ in range(nranks)]          # [owner][source]
    flags = [[[0] * nranks for _ in range(ncta)] for _ in range(nranks)]
    launch = [0] * nranks
    ctas = [[{"pc": "vote", "row": b} for b in range(ncta)] for _ in range(nranks)]
    steps = 0
    while any(x < nlaunches for x in launch):
        steps += 1
        assert steps < 200_000
        runnable = []
        for r in range(nranks):
            if launch[r] >= nlaunches:
                continue
            e1, e2 = 2 * launch[r] + 1, 2 * launch[r] + 2
            for i, cta in enumerate(ctas[r]):
                need = e1 if cta["pc"] == "wait1" else e2 if cta["pc"] == "wait2" else None
                if need is not None and not all(flags[r][cta["row"]][p] >= need for p in range(nranks)):
                    continue
                if cta["pc"] != "done":
                    runnable.append((r, i))
        r, i = rng.choice(runnable)
        cta, c = ctas[r][i], launch[r]
        if cta["pc"] == "vote":
            for p in range(nranks):
                votes[p][r] = (r, c)
            cta["pc"] = "arrive1"
        elif cta["pc"] == "arrive1":
            for p in range(nranks):
                flags[p][cta["row"]][r] = 2 * c + 1
            cta["pc"] = "wait1"
        elif cta["pc"] == "wait1":
            cta["pc"] = "read"
        elif cta["pc"] == "read":
            for p in range(nranks):
                if votes[r][p] != (p, c):
                    return f"rank {r} launch {c} row {cta['row']} read vote {votes[r][p]} of rank {p}"
            cta["pc"] = "arrive2" if closing_barrier else "done"
        elif cta["pc"] == "arrive2":
            for p in range(nranks):
                flags[p][cta["row"]][r] = 2 * c + 2
            cta["pc"] = "wait2"
        elif cta["pc"] == "wait2":
            cta["pc"] = "done"
        if all(x["pc"] == "done" for x in ctas[r]):
            launch[r] += 1
            ctas[r] = [{"pc": "vote", "row": b} for b in range(ncta)]
    return None


def test_single_vote_area_is_safe_because_of_the_closing_barrier():
    for seed in range(300):
        rng = random.Random(seed)
        assert run_vote_schedule(rng.randint(2, 3), rng.randint(1, 3), 4, rng, closing_barrier=True) is None


def test_single_vote_area_would_race_without_the_closing_barrier():
    """Why the comment in peer.cuh insists on it: with more than one CTA per rank and no closing barrier, a rank whose rows have all
    passed the vote barrier can start the next launch and overwrite its word before a peer's slower ROW has read it."""
    found = None
    for seed in range(300):
        rng = random.Random(seed)
        found = found or run_vote_schedule(2, 2, 4, rng, closing_barrier=False)
    assert found is not None
