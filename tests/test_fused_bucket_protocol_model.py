"""Schedule-exploring model of ``allreduce_update_kernel`` (bagua_b200/csrc/peer_kernels.cu): one launch per
bucket does  barrier → reduce-scatter (rank r pulls slice r of every peer's gradient bucket) → optimizer step on the slice →
all-gather (pushes the new weights of slice r into every peer's weight bucket) → barrier → zero the own gradient bucket.

All barriers are per CTA ROW.  That is enough only because the work is column-striped: CTA b of every rank touches column range b
of every slice — in the pull, in the push and in the zeroing — so "row b of every peer has passed the barrier" is exactly "everything
I am about to overwrite has been read" (``walk_owned_slice`` and ``for_each_striped``; comment at the gradient clear of the kernel).  The model runs random interleavings of the CTAs
of 2-3 ranks over several steps, with backward writing fresh gradients between launches, and checks every value read; zeroing
without the column discipline must be caught."""
import random

import pytest


def run(nranks, ncta, steps, rng, striped_zeroing=True):
    ncol = ncta                                   # one cell per (slice, column range)
    grads = [[[("g", r, 0)] * ncol for _ in range(nranks)] for r in range(nranks)]     # [owner][slice][col] = ("g", producer, step) or 0
    weights = [[[None] * ncol for _ in range(nranks)] for _ in range(nranks)]          # [owner][slice][col] = step of the update
    flags = [[[0] * nranks for _ in range(ncta)] for _ in range(nranks)]
    step_of = [0] * nranks
    program = ["arrive1", "wait1", "pull_update_push", "arrive2", "wait2", "zero"]

    def fresh():
        return [{"ip": 0} for _ in range(ncta)]

    ctas = [fresh() for _ in range(nranks)]
    guard = 0
    while any(s < steps for s in step_of):
        guard += 1
        assert guard < 300_000
        runnable = []
        for r in range(nranks):
            if step_of[r] >= steps:
                continue
            for b, cta in enumerate(ctas[r]):
                if cta["ip"] >= len(program):
                    continue
                op = program[cta["ip"]]
                if op in ("wait1", "wait2"):
                    need = 2 * step_of[r] + (1 if op == "wait1" else 2)
                    if not all(flags[r][b][p] >= need for p in range(nranks)):
                        continue
                runnable.append((r, b))
        r, b = rng.choice(runnable)
        cta, c = ctas[r][b], step_of[r]
        op = program[cta["ip"]]
        if op in ("arrive1", "arrive2"):
            for p in range(nranks):
                flags[p][b][r] = 2 * c + (1 if op == "arrive1" else 2)
        elif op == "pull_update_push":
            for p in range(nranks):              # my slice r, my column b, from every peer's gradient bucket
                if grads[p][r][b] != ("g", p, c):
                    return f"step {c}: rank {r} row {b} pulled {grads[p][r][b]} from rank {p} (expected its step-{c} gradient)"
            for p in range(nranks):              # the updated weights of slice r, column b → everybody
                weights[p][r][b] = c
        elif op == "zero":
            cols = [b] if striped_zeroing else range(ncol)
            for s in range(nranks):
                for col in cols:
                    grads[r][s][col] = 0
        cta["ip"] += 1
        if all(x["ip"] >= len(program) for x in ctas[r]):
            # the kernel has retired: the trainer reads the gathered weights, then the next backward accumulates into the zeroed bucket
            for s in range(nranks):
                for col in range(ncol):
                    if weights[r][s][col] != c:
                        return f"step {c}: rank {r} sees weights of slice {s} column {col} from step {weights[r][s][col]}"
                    if grads[r][s][col] != 0:
                        return f"step {c}: rank {r} starts the next backward on a gradient cell that was not cleared"
                    grads[r][s][col] = ("g", r, c + 1)
            step_of[r] += 1
            ctas[r] = fresh()
    return None


@pytest.mark.parametrize("nranks,ncta", [(2, 1), (2, 3), (3, 2)])
def test_column_striping_makes_per_row_barriers_sufficient(nranks, ncta):
    for seed in range(150):
        assert run(nranks, ncta, steps=3, rng=random.Random(seed)) is None


def test_zeroing_outside_the_own_column_range_is_caught():
    found = None
    for seed in range(300):
        found = found or run(2, 3, steps=2, rng=random.Random(seed), striped_zeroing=False)
    assert found is not None and "pulled" in found
