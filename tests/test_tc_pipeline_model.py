"""A small executable model of the wgmma linear kernel's synchronisation (csrc/cuda/tc_gemm.cu): the TMA producer and the
two consumer warpgroups, the shared-memory ring that runs through tile boundaries, the asynchronous MMA groups (a stage
is released only once the group that reads it has completed: one group stays in flight), and the exact parity
expressions the kernel passes to its mbarrier waits.  mbarriers are modelled with their phase semantics
(``try_wait.parity(P)`` succeeds once the phase of parity P has completed).  A random scheduler interleaves the roles;
the model asserts what the hardware would silently get wrong:

* a ring stage is never refilled before both warpgroups released it, nor while an MMA group still reads it,
* an MMA never reads a stage that has not been filled for this k-block,
* nobody dead-locks, and every tile comes out of both warpgroups with the right (tile, k-block) contributions.

The kernel itself cannot run here (no GPU); this guards the protocol when the loops are edited."""
import random

import pytest


class MBar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):
        return self.phase != parity


def run_model(n_tiles, grid, cta, nkb, stages, seed, consumers=2, bug=None):
    """One CTA of the persistent kernel.  Roles are generators that yield while blocked or between steps."""
    rng = random.Random(seed)
    full = [MBar(1) for _ in range(stages)]
    empty = [MBar(consumers) for _ in range(stages)]
    ring = [None] * stages              # (tile, kblock) currently in the stage
    need = [set() for _ in range(stages)]       # warpgroups that have not released the stage yet
    reading = [set() for _ in range(stages)]    # warpgroups whose issued MMA group on the stage has not completed
    results = {}
    my_tiles = list(range(cta, n_tiles, grid))

    def producer():
        g = 0
        for t in my_tiles:
            for i in range(nkb):
                s, rnd = g % stages, g // stages
                if rnd > 0 and bug != "producer_never_waits":
                    while not empty[s].passed((rnd & 1) if bug == "producer_parity" else ((rnd - 1) & 1)):
                        yield
                assert not need[s], f"stage {s} refilled while ({ring[s]}) is unread by {need[s]}"
                assert not reading[s], f"stage {s} refilled while an MMA group of {reading[s]} still reads it"
                ring[s] = (t, i)
                need[s] = set(range(consumers))
                full[s].arrive()            # arrive.expect_tx + the TMA bytes landing
                g += 1
                yield

    def release(c, s):
        need[s].discard(c)
        empty[s].arrive()

    def consumer(c):
        g = 0
        for t in my_tiles:
            ks, prev = [], None
            for i in range(nkb):
                s = g % stages
                while not full[s].passed((g // stages) & 1):
                    yield
                assert ring[s] == (t, i), f"MMA of warpgroup {c} for ({t},{i}) found {ring[s]} in stage {s}"
                assert c in need[s], f"warpgroup {c} reads stage {s} twice"
                reading[s].add(c)           # wgmma.mma_async x 4 + commit_group
                ks.append(i)
                if bug == "consumer_releases_early":
                    release(c, s)
                yield
                if prev is not None:        # wgmma.wait_group 1: the previous stage's group has completed
                    reading[prev].discard(c)
                    if bug != "consumer_releases_early":
                        release(c, prev)
                prev = s
                g += 1
                yield
            reading[prev].discard(c)        # wgmma.wait_group 0
            if bug != "consumer_releases_early":
                release(c, prev)
            results[(t, c)] = ks
            yield                           # the epilogue from registers

    roles = [producer()] + [consumer(c) for c in range(consumers)]
    live = list(roles)
    idle_rounds = 0
    while live:
        r = rng.choice(live)
        before = (tuple(b.phase for b in full + empty), tuple(b.pending for b in empty), len(results))
        try:
            next(r)
        except StopIteration:
            live.remove(r)
            idle_rounds = 0
            continue
        after = (tuple(b.phase for b in full + empty), tuple(b.pending for b in empty), len(results))
        idle_rounds = idle_rounds + 1 if before == after else 0
        assert idle_rounds < 20000, "dead-lock: no role made progress"
    assert sorted(results) == sorted((t, c) for t in my_tiles for c in range(consumers))
    for k, v in results.items():
        assert v == list(range(nkb)), f"tile/warpgroup {k} accumulated {v}"
    return len(my_tiles)


@pytest.mark.parametrize("n_tiles,grid,nkb,stages", [
    (1, 1, 1, 6), (1, 1, 13, 5), (5, 1, 1, 6), (5, 1, 3, 5), (7, 2, 8, 6), (9, 4, 2, 5), (16, 3, 6, 6), (4, 4, 20, 5),
    (33, 8, 1, 2), (12, 5, 7, 3),
])
def test_pipeline_protocol_under_random_interleavings(n_tiles, grid, nkb, stages):
    done = 0
    for cta in range(grid):
        for seed in range(6):
            n = run_model(n_tiles, grid, cta, nkb, stages, seed * 977 + cta)
        done += n
    assert done == n_tiles          # the CTAs of a launch cover every tile exactly once


@pytest.mark.parametrize("bug", ["producer_parity", "producer_never_waits", "consumer_releases_early"])
def test_model_catches_protocol_bugs(bug):
    """Sanity of the model itself: a wrong parity or a missing wait must trip an assertion (or the dead-lock check)
    in at least one interleaving."""
    caught = 0
    for seed in range(40):
        try:
            run_model(12, 2, 0, 5, 3, seed, bug=bug)
        except AssertionError:
            caught += 1
    assert caught > 0
