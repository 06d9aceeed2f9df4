"""Schedule-exploring model of the overflow vote of the in-bucket optimizers with loss scaling (``loss_scale_norm_kernel`` and the
phase-B kernels that obey it, bagua_b200/csrc/peer_kernels.cu):

    exchange (once per step)   publish my Σx² into slot [half][r] of every peer's box → barrier → read slots [half][0..P) in rank order
                               → {total, coef, found_inf}; t += !found_inf
    phase B (per step)         read {coef, found_inf, t}; skipped: nothing; taken: push the weights of slice r to every peer; → barrier
    trainer                    reads every slice of its weights, then the next step begins

The box is the double-buffered one of ``tests/test_clip_norm_protocol_model.py`` (the half alternates with the op's call counter, no
closing barrier). Random interleavings of the ranks are explored over several steps in which some rank's sum is non-finite. Checked:
every rank reads this step's sums of all ranks, so all three words and the step count agree on every rank; the skip / take decision
is therefore uniform and the phase-B barriers stay matched (the model would deadlock otherwise); a skipped step leaves every weight
slice at the version of the last taken step. The exchange must not lean on the barrier of the kernel that happens to follow it: run
back to back on its own (``phase_b=False``, as the kernel tests launch it) the double-buffered box is still safe, and the
single-buffered box without a closing barrier is caught."""
import math
import random

import pytest


def local_sum(r, c, overflow):
    return math.inf if overflow.get(c) == r else float(1 + r + 10 * c)


def run(nranks, steps, rng, overflow, double_buffer=True, phase_b=True):
    box = [[[None] * nranks for _ in range(2)] for _ in range(nranks)]   # [owner][half][slot]
    weights = [[0] * nranks for _ in range(nranks)]                      # [owner][slice] = t of the update that wrote it
    flags = [[0] * nranks for _ in range(nranks)]
    epoch, ncalls, t = [0] * nranks, [0] * nranks, [0] * nranks
    vote = [None] * nranks
    votes = [dict() for _ in range(steps)]
    prog = ["N.pub", "N.arrive", "N.wait", "N.read"] + (["B.update", "B.arrive", "B.wait", "trainer"] if phase_b else [])
    step_of, ip = [0] * nranks, [0] * nranks
    guard = 0
    while any(s < steps for s in step_of):
        guard += 1
        assert guard < 200_000
        runnable = [r for r in range(nranks) if step_of[r] < steps
                    and not (prog[ip[r]].endswith(".wait") and not all(flags[r][p] >= epoch[r] for p in range(nranks)))]
        assert runnable, "deadlock: the ranks disagree on which barriers to take"
        r = rng.choice(runnable)
        c, op = step_of[r], prog[ip[r]]
        half = (ncalls[r] & 1) if double_buffer else 0
        if op.endswith(".arrive"):
            epoch[r] += 1
            for p in range(nranks):
                flags[p][r] = epoch[r]
        elif op == "N.pub":
            for p in range(nranks):
                box[p][half][r] = (c, local_sum(r, c, overflow))
        elif op == "N.read":
            got = box[r][half]
            if [g[0] for g in got] != [c] * nranks:
                return f"step {c}: rank {r} read the sums of steps {[g[0] for g in got]}"
            S = 0.0
            for _, v in got:   # rank order
                S += v
            found = not math.isfinite(S)
            t[r] += 0 if found else 1
            vote[r] = (math.sqrt(S), min(1.0 / (math.sqrt(S) + 1e-6), 1.0), found, t[r])
            votes[c][r] = vote[r]
            ncalls[r] += 1
        elif op == "B.update":
            if not vote[r][2]:
                for p in range(nranks):
                    weights[p][r] = vote[r][3]
        elif op == "trainer":
            if weights[r] != [t[r]] * nranks:
                return f"step {c}: rank {r} reads weights of versions {weights[r]}, its step count is {t[r]}"
        ip[r] += 1
        if ip[r] == len(prog):
            step_of[r] += 1
            ip[r] = 0
    for c, v in enumerate(votes):
        if len(set(v.values())) != 1:
            return f"step {c}: the ranks voted differently: {v}"
        if next(iter(v.values()))[2] != (c in overflow):
            return f"step {c}: wrong vote {v}"
    taken = steps - len(overflow)
    if t != [taken] * nranks:
        return f"step counts {t}, expected {taken} everywhere"
    return None


OVERFLOW = {0: 1, 3: 0}   # step → the rank whose sum is non-finite: the very first step, and a later one


@pytest.mark.parametrize("phase_b", [True, False])
@pytest.mark.parametrize("nranks", [2, 3, 4])
def test_every_rank_reads_the_same_vote(nranks, phase_b):
    for seed in range(200):
        assert run(nranks, steps=6, rng=random.Random(seed), overflow=OVERFLOW, phase_b=phase_b) is None


def test_single_buffered_box_is_caught():
    found = None
    for seed in range(400):
        found = found or run(2, steps=6, rng=random.Random(seed), overflow=OVERFLOW, double_buffer=False, phase_b=False)
    assert found is not None and ("read the sums" in found or "voted differently" in found), found
