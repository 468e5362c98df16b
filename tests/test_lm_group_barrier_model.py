"""Host model of the group barrier of the batched k_lm_persistent (ct_icp_b200/csrc/icp_lm.cu, lm_group_barrier).

A batched launch runs B registrations; group g owns the CTAs [first_cta[g], first_cta[g + 1]): the first is its solver
CTA, the others its workers. Where the solo kernel separates its phases with grid.sync(), a grouped CTA calls the group
barrier: thread 0 adds 1 to the group's counter (zeroed before every launch) and polls it until it reaches
barrier_index * group_ctas. The wait is bounded: a CTA that has waited too long sets the group's abort word, and a
waiter that finds the abort word set leaves too; the solver CTA then marks the group's state failed = 2.

Each CTA below is a real thread that runs the LM loop's own phase sequence (initial barrier; per ICP iteration: residual
assembly, barrier, GetProblem, barrier, then per LM evaluation: evaluation, barrier, minimizer step, barrier), with the
`st->done` / `lm->done` breaks read from the group's state after a barrier, as in the kernel. Each group follows its own
script (ICP iterations until convergence, evaluations per solve, a failure at GetProblem), so groups take different
numbers of barriers. Checked: no group's progress depends on another's, every thread exits after convergence, failure and
a time-out, a time-out leaves the other groups' results unchanged, and the worker-to-partial-row mapping and the solver's
reduction order are those of the solo kernel with the same worker count."""
import random
import threading
import time

import numpy as np
import pytest

K_ACC = 96          # kAcc
K_LMP_WARPS = 16    # kLmPWarps
K_IN_FLIGHT = 10    # the solver's rows in flight per warp (k_lm_persistent's reduction)
TIMEOUT_S = 0.4     # kLoopSyncTimeout, scaled to the model


class Barriers:
    """the barrier words of a launch: per group an arrival counter and an abort word (zeroed before every launch)"""

    def __init__(self, groups):
        self.lock = threading.Lock()
        self.count = [0] * groups
        self.abort = [0] * groups

    def zero(self):
        with self.lock:
            self.count = [0] * len(self.count)
            self.abort = [0] * len(self.abort)

    def arrive_and_wait(self, g, target, stall=None):
        """lm_group_barrier's thread 0: atomicAdd, then poll (acquire) until target, the abort word or the time-out"""
        if stall is not None:
            stall.wait()                 # a CTA held up before it arrives
        with self.lock:
            self.count[g] += 1
        t0 = time.monotonic()
        while True:
            with self.lock:
                if self.count[g] >= target:
                    return True
                if self.abort[g]:
                    return False
            if time.monotonic() - t0 > TIMEOUT_S:
                with self.lock:
                    self.abort[g] = 1
                return False
            time.sleep(0.0005 * random.random())


class GroupState:
    """what the group's CTAs share through global memory: IcpState.done / failed, LmState.done, the trace of phases"""

    def __init__(self, script):
        self.script = script         # dict: icp_iters (until convergence), evals (per solve), fail_at_select
        self.st_done = 0
        self.failed = 0
        self.lm_done = 0
        self.iters = 0
        self.evaluations = 0
        self.barriers = {}           # cta -> barriers taken
        self.phases = []             # the solver's phase log


def run_cta(bar, g, cta, group_ctas, S, num_iters_icp, ls_max_num_iters, stall=None):
    """one CTA of group g: the phase sequence of lm_persistent_body (kGrouped)"""
    solver = cta == 0
    taken = 0

    def sync():
        nonlocal taken
        taken += 1
        return bar.arrive_and_wait(g, taken * group_ctas, stall if taken == 3 else None)

    time.sleep(0.001 * random.random())
    live = sync()
    it = 0
    while live and it < num_iters_icp:
        if S.st_done:
            break
        time.sleep(0.0005 * random.random())            # residual assembly (workers)
        if not sync():
            live = False
            break
        if solver:                                       # GetProblem
            S.phases.append(("select", it))
            if S.script.get("fail_at_select") == it:
                S.failed, S.st_done, S.lm_done = 1, 1, 1
            else:
                S.lm_done = 0
        if not sync():
            live = False
            break
        for ev in range(ls_max_num_iters + 1):
            if S.st_done or S.lm_done:
                break
            time.sleep(0.0003 * random.random())        # evaluation (workers)
            if not sync():
                live = False
                break
            if solver:                                   # minimizer step; the solve ends after script["evals"]
                S.evaluations += 1
                S.phases.append(("step", it, ev))
                if ev + 1 >= S.script["evals"] or ev == ls_max_num_iters:
                    S.lm_done = 1
                    S.iters = it + 1
                    if it + 1 >= S.script["icp_iters"]:
                        S.st_done = 1
            if not sync():
                live = False
                break
        if not live:
            break
        it += 1
    if solver and not live:
        S.failed, S.st_done = 2, 1
    S.barriers[cta] = taken


def launch(bar, scripts, group_ctas, num_iters_icp=6, ls_max_num_iters=5, stalled=None, deadline=10.0):
    """one batched launch: returns the groups' states and the threads; `stalled` = (group, cta, event)"""
    bar.zero()
    states = [GroupState(s) for s in scripts]
    threads = []
    for g, n in enumerate(group_ctas):
        for cta in range(n):
            stall = stalled[2] if stalled and stalled[:2] == (g, cta) else None
            t = threading.Thread(target=run_cta, args=(bar, g, cta, n, states[g], num_iters_icp, ls_max_num_iters, stall),
                                 daemon=True)
            threads.append((g, cta, t))
    for _, _, t in threads:
        t.start()
    return states, threads


def join(threads, groups=None, deadline=10.0):
    end = time.monotonic() + deadline
    for g, _, t in threads:
        if groups is None or g in groups:
            t.join(max(0.0, end - time.monotonic()))
    return all(not t.is_alive() for g, _, t in threads if groups is None or g in groups)


SCRIPTS = [
    {"icp_iters": 1, "evals": 2},                   # converged after its first ICP iteration
    {"icp_iters": 99, "evals": 6},                  # runs every iteration, every evaluation
    {"icp_iters": 99, "evals": 1, "fail_at_select": 0},   # too few residuals: fails at GetProblem
    {"icp_iters": 3, "evals": 3},
]
CTAS = [3, 5, 2, 4]


def _result(S):
    return (S.st_done, S.failed, S.iters, S.evaluations, tuple(S.phases))


def _solo(script, ctas):
    bar = Barriers(1)
    (S,), threads = launch(bar, [script], [ctas])
    assert join(threads)
    return _result(S)


def test_groups_with_different_barrier_counts_finish_independently():
    solo = [_solo(s, n) for s, n in zip(SCRIPTS, CTAS)]
    bar = Barriers(len(SCRIPTS))
    for _ in range(2):                                  # two launches: the counters are zeroed in between
        states, threads = launch(bar, SCRIPTS, CTAS)
        assert join(threads), "a thread did not exit"
        assert [_result(S) for S in states] == solo
        counts = [set(S.barriers.values()) for S in states]
        assert all(len(c) == 1 for c in counts), counts          # every CTA of a group took the same barriers
        assert len({next(iter(c)) for c in counts}) == len(SCRIPTS)   # and the groups took different numbers
        assert [S.failed for S in states] == [0, 0, 1, 0]


def test_a_stalled_cta_times_out_its_group_alone():
    solo = [_solo(s, n) for s, n in zip(SCRIPTS, CTAS)]
    bar = Barriers(len(SCRIPTS))
    hold = threading.Event()
    states, threads = launch(bar, SCRIPTS, CTAS, stalled=(1, 2, hold))   # worker 2 of group 1 stops before barrier 3
    others = {0, 2, 3}
    assert join(threads, others), "another group waited for the stalled one"
    assert [_result(states[g]) for g in sorted(others)] == [solo[g] for g in sorted(others)]
    assert join(threads, {1}, deadline=5 * TIMEOUT_S) is False     # the stalled thread itself is still held
    time.sleep(2 * TIMEOUT_S)
    assert states[1].failed == 2 and states[1].st_done == 1
    hold.set()                                          # the late CTA arrives, finds the abort word and leaves
    assert join(threads), "a thread of the timed-out group did not exit"
    # the next launch zeroes the words: the same group runs normally again
    states, threads = launch(bar, SCRIPTS, CTAS)
    assert join(threads)
    assert [_result(S) for S in states] == solo


def _solver_reduce(partials, first_row, workers):
    """k_lm_persistent's reduction: warp w sums rows w, w + 16, … in chunks of K_IN_FLIGHT, then the per-warp sums in order"""
    part = np.zeros((K_LMP_WARPS, K_ACC))
    for w in range(K_LMP_WARPS):
        a = np.zeros(K_ACC)
        for b0 in range(w, workers, K_LMP_WARPS * K_IN_FLIGHT):
            for u in range(K_IN_FLIGHT):
                b = b0 + u * K_LMP_WARPS
                if b < workers:
                    a = a + partials[first_row + b]
        part[w] = a
    s = np.zeros(K_ACC)
    for w in range(K_LMP_WARPS):
        s = s + part[w]
    return s


@pytest.mark.parametrize("gathers", [[2, 30, 29, 28], [1, 1, 1], [131], [40, 1, 65, 7]])
def test_partial_rows_and_reduction_order_match_the_solo_kernel(gathers):
    rng = np.random.default_rng(len(gathers))
    first_cta = np.concatenate([[0], np.cumsum([1 + n for n in gathers])])
    rows = np.zeros((first_cta[-1] - len(gathers), K_ACC))
    solo_rows = []
    for g, n in enumerate(gathers):
        vals = rng.standard_normal((n, K_ACC)) * 10.0 ** rng.integers(-8, 8, size=(n, 1))
        solo_rows.append(vals)
        for cta in range(first_cta[g], first_cta[g + 1]):
            c = cta - first_cta[g]
            if c == 0:
                continue                                # the solver CTA writes no row
            row = (first_cta[g] - g) + (c - 1)          # partials + (first_cta[g] - g) * kAcc + wi * kAcc
            assert not rows[row].any(), "two workers on one row"
            rows[row] = vals[c - 1]
    assert np.count_nonzero(np.abs(rows).sum(axis=1)) == rows.shape[0]   # every row written
    for g, n in enumerate(gathers):
        grouped = _solver_reduce(rows, first_cta[g] - g, n)
        solo = _solver_reduce(solo_rows[g], 0, n)
        assert grouped.tobytes() == solo.tobytes()
