"""Schedule-exploring model of the per-parameter ratio exchange of the in-bucket LAMB (``lamb_ratio_kernel``, peer_kernels.cu):

    ratio exchange (step())   write my (Σw², Σu²) of every parameter into slot [half][r] of every peer's box → barrier →
                              read slots [half][0..P) of every parameter, in rank order
    apply (per bucket)        read the ratios → update the shard → push the weights of slice r to every peer → (closing barrier)
    trainer                   reads every slice of its weights (next forward)

Each rank runs its kernels in stream order; random interleavings of the ranks are explored over several steps. Checked: every rank
reads this call's sums from every peer, for every parameter, and the trainer sees this step's weights. The exchange must not rely
on the barriers around it, so the model can also drop the apply kernel's closing barrier: the box half alternates with the op's
call counter, and that alone keeps the exchange safe; a single-buffered box without a closing barrier must be caught."""
import random

import pytest


def run(nranks, nparams, steps, rng, double_buffer=True, closing_barrier=False, apply_barrier=True):
    box = [[[[None] * nparams for _ in range(nranks)] for _ in range(2)] for _ in range(nranks)]   # [owner][half][slot][param]
    weights = [[None] * nranks for _ in range(nranks)]
    flags = [[0] * nranks for _ in range(nranks)]
    epoch = [0] * nranks
    ratio = [None] * nranks
    calls = [0] * nranks

    def program():
        prog = ["R.pub", "R.arrive", "R.wait", "R.read"] + (["R.arrive", "R.wait"] if closing_barrier else [])
        return prog + ["B.push"] + (["B.arrive", "B.wait"] if apply_barrier else []) + ["trainer"]

    step_of, ip = [0] * nranks, [0] * nranks
    prog = program()
    guard = 0
    while any(s < steps for s in step_of):
        guard += 1
        assert guard < 200_000
        runnable = [r for r in range(nranks) if step_of[r] < steps and not (
            prog[ip[r]].endswith(".wait") and not all(flags[r][p] >= epoch[r] for p in range(nranks)))]
        r = rng.choice(runnable)
        c, op = step_of[r], prog[ip[r]]
        half = (calls[r] & 1) if double_buffer else 0
        if op.endswith(".arrive"):
            epoch[r] += 1
            for p in range(nranks):
                flags[p][r] = epoch[r]
        elif op == "R.pub":
            for p in range(nranks):
                for t in range(nparams):   # the kernel's threads store parameter by parameter: a reader may see a partial write
                    box[p][half][r][t] = (r, c, t)
        elif op == "R.read":
            for t in range(nparams):
                got = [box[r][half][p][t] for p in range(nranks)]
                want = [(p, c, t) for p in range(nranks)]
                if got != want:
                    return f"step {c}: rank {r} ratio call {calls[r]} read {got} for parameter {t}, expected {want}"
            ratio[r] = c
            calls[r] += 1
        elif op == "B.push":
            if ratio[r] != c:
                return f"step {c}: rank {r} applies the ratios of step {ratio[r]}"
            for p in range(nranks):
                weights[p][r] = c
        elif op == "trainer":
            if apply_barrier:
                for s in range(nranks):
                    if weights[r][s] != c:
                        return f"step {c}: rank {r} reads weights of slice {s} from step {weights[r][s]}"
        ip[r] += 1
        if ip[r] == len(prog):
            step_of[r] += 1
            ip[r] = 0
    return None


@pytest.mark.parametrize("nranks", [2, 3, 4])
def test_double_buffered_ratio_box_is_safe(nranks):
    for seed in range(200):
        assert run(nranks, 3, steps=4, rng=random.Random(seed)) is None
        assert run(nranks, 3, steps=4, rng=random.Random(seed), apply_barrier=False) is None


def test_single_buffered_box_with_a_closing_barrier_is_safe():
    for seed in range(200):
        assert run(3, 3, steps=4, rng=random.Random(seed), double_buffer=False, closing_barrier=True, apply_barrier=False) is None


def test_single_buffered_box_without_closing_barrier_is_caught():
    found = None
    for seed in range(400):
        found = found or run(2, 3, steps=4, rng=random.Random(seed), double_buffer=False, apply_barrier=False)
    assert found is not None and "ratio call" in found
