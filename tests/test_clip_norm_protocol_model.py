"""Schedule-exploring model of global-norm clipping in the in-bucket optimizers (bagua_b200/csrc/peer_kernels.cu):

    phase A (per bucket, in backward)   barrier → pull slice r of every peer's gradient bucket → fp32 shard + partial Σx² → barrier → clear
    norm exchange (step(), or clip_grad_norm_ before it; a user may call it more than once per step)
                                        publish my Σ into slot [half][r] of every peer's box → barrier → read slots [half][0..P)
    phase B (per bucket, in step())     read coef → update the shard → push the weights of slice r to every peer → barrier
    trainer                             reads every slice of its weights (next forward), then backward refills the bucket

Each rank runs its kernels in stream order; random interleavings of the ranks are explored over several steps. Checked: phase A
pulls this step's gradients, every norm read sees this call's sums of all ranks (so phase B applies this step's coefficient), and the
trainer sees this step's weights.  The box half alternates with a host call counter; a single-buffered box without a closing
barrier, and phase B without its closing barrier, must be caught."""
import random

import pytest


def run(nranks, steps, rng, double_buffer=True, norm_closing_barrier=False, b_barrier=True):
    calls_per_step = [rng.choice((1, 2)) for _ in range(steps)]   # every rank issues the same norm calls
    grads = [[("g", r, 0)] * nranks for r in range(nranks)]       # [owner][slice]
    weights = [[None] * nranks for _ in range(nranks)]             # [owner][slice] = step of the update
    box = [[[None] * nranks for _ in range(2)] for _ in range(nranks)]   # [owner][half][slot]
    flags = [[0] * nranks for _ in range(nranks)]                  # flags[owner][from] = epoch
    epoch = [0] * nranks
    coef = [None] * nranks
    ncalls = [0] * nranks

    def program(c):
        prog = ["A.arrive", "A.wait", "A.pull", "A.arrive", "A.wait", "A.zero"]
        for _ in range(calls_per_step[c]):
            prog += ["N.pub", "N.arrive", "N.wait", "N.read"] + (["N.arrive", "N.wait"] if norm_closing_barrier else [])
        prog += ["B.push"] + (["B.arrive", "B.wait"] if b_barrier else []) + ["trainer"]
        return prog

    step_of = [0] * nranks
    ip = [0] * nranks
    progs = [program(0) for _ in range(nranks)]
    guard = 0
    while any(s < steps for s in step_of):
        guard += 1
        assert guard < 200_000
        runnable = []
        for r in range(nranks):
            if step_of[r] >= steps:
                continue
            op = progs[r][ip[r]]
            if op.endswith(".wait") and not all(flags[r][p] >= epoch[r] for p in range(nranks)):
                continue
            runnable.append(r)
        r = rng.choice(runnable)
        c, op = step_of[r], progs[r][ip[r]]
        half = (ncalls[r] & 1) if double_buffer else 0
        if op.endswith(".arrive"):
            epoch[r] += 1
            for p in range(nranks):
                flags[p][r] = epoch[r]
        elif op == "A.pull":
            for p in range(nranks):
                if grads[p][r] != ("g", p, c):
                    return f"step {c}: rank {r} pulled {grads[p][r]} from rank {p}"
        elif op == "A.zero":
            grads[r] = [0] * nranks
        elif op == "N.pub":
            for p in range(nranks):
                box[p][half][r] = (r, c, ncalls[r])
        elif op == "N.read":
            got = box[r][half]
            want = [(p, c, ncalls[r]) for p in range(nranks)]
            if got != want:
                return f"step {c}: rank {r} norm call {ncalls[r]} read {got}, expected {want}"
            coef[r] = (c, ncalls[r])
            ncalls[r] += 1
        elif op == "B.push":
            if coef[r] is None or coef[r][0] != c:
                return f"step {c}: rank {r} phase B applies the coefficient of {coef[r]}"
            for p in range(nranks):
                weights[p][r] = c
        elif op == "trainer":
            for s in range(nranks):
                if weights[r][s] != c:
                    return f"step {c}: rank {r} reads weights of slice {s} from step {weights[r][s]}"
            grads[r] = [("g", r, c + 1)] * nranks       # backward of the next step refills the (cleared) bucket
        ip[r] += 1
        if ip[r] == len(progs[r]):
            step_of[r] += 1
            ip[r] = 0
            if step_of[r] < steps:
                progs[r] = program(step_of[r])
    return None


@pytest.mark.parametrize("nranks", [2, 3, 4])
def test_double_buffered_norm_box_is_safe(nranks):
    for seed in range(200):
        assert run(nranks, steps=4, rng=random.Random(seed)) is None


def test_single_buffered_box_with_a_closing_barrier_is_safe():
    for seed in range(200):
        assert run(3, steps=4, rng=random.Random(seed), double_buffer=False, norm_closing_barrier=True) is None


def test_single_buffered_box_without_closing_barrier_is_caught():
    found = None
    for seed in range(400):
        found = found or run(2, steps=4, rng=random.Random(seed), double_buffer=False)
    assert found is not None and "norm call" in found


def test_phase_b_without_closing_barrier_is_caught():
    found = None
    for seed in range(400):
        found = found or run(2, steps=3, rng=random.Random(seed), b_barrier=False)
    assert found is not None and "reads weights" in found
