"""Synchronisation of one conv_c8_kernel CTA with one or two teams of ping-pong warpgroups, as a discrete model.

The model is written from the protocol of se_conv_c8.cu (DESIGN.md 5.1), not from its code: a producer that loads one halo
per tile into a ring of buffers (an mbarrier pair per buffer: `full`, one arrival by the load; `empty`, one arrival per
reading warpgroup here, per warp in the kernel), TEAMS x 2 consumer warpgroups, team t running the CTA's tiles t,
t + TEAMS, ... and all `ncls` classes of each, and per team two named barriers that order the warpgroups' MMA issue:
warpgroup 0 arrives on the first for every virtual tile, where warpgroup 1 syncs; warpgroup 1 arrives on the second for
every virtual tile but its last, where warpgroup 0 syncs for every one but its first.

Actors run under seeded random interleavings. A run must terminate; every (tile, class, warpgroup) is computed once, from
the buffer the producer filled for that tile; no buffer is refilled before both its readers released it; within a team
the issue order is wg0(v), wg1(v), wg0(v + 1), ...; and every named barrier ends with no pending arrival. A hang or a
half-arrived barrier on a GPU is found here instead.
"""
import random

import pytest


class Violation(Exception):
    pass


class MBar:
    """mbarrier: `count` arrivals complete a phase; wait(parity) passes once the phase of that parity has completed."""

    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):
        return self.phase != parity


class NamedBar:
    """bar.sync / bar.arrive over two warpgroups: the second arrival completes a generation and resets the barrier."""

    def __init__(self):
        self.count, self.gen = 0, 0

    def arrive(self):
        self.count += 1
        if self.count == 2:
            self.count, self.gen = 0, self.gen + 1


def ring_of(i, n):
    return i % n, (i // n) & 1


def simulate(tiles, ncls, depth, teams, seed, skip_last_arrive=True, shared_ids=False):
    full = [MBar(1) for _ in range(depth)]
    empty = [MBar(2) for _ in range(depth)]
    bars = {}
    held = [None] * depth        # tile whose halo the buffer holds
    readers = [0] * depth        # warpgroups that have not released it yet
    computed = {}
    issued = [[0, 0] for _ in range(teams)]   # virtual tiles issued so far, per team and warpgroup

    def bar(team, which):        # which = 0: where warpgroup 1 waits; 1: where warpgroup 0 waits
        return bars.setdefault(1 + which + (0 if shared_ids else 2 * team), NamedBar())

    def producer():
        for riter in range(tiles):
            slot, ph = ring_of(riter, depth)
            yield lambda: empty[slot].passed(ph ^ 1)
            if readers[slot]:
                raise Violation("buffer %d refilled for tile %d while tile %s is still read" % (slot, riter, held[slot]))
            held[slot], readers[slot] = riter, 2
            yield lambda: True   # the load is in flight
            full[slot].arrive()

    def warpgroup(team, wg):
        nv = len(range(team, tiles, teams)) * ncls
        for v in range(nv):
            riter, cls = team + (v // ncls) * teams, v % ncls
            slot, ph = ring_of(riter, depth)
            yield lambda: full[slot].passed(ph)
            if wg == 1 or v > 0:
                b = bar(team, 1 - wg)
                gen = b.gen
                b.arrive()
                yield lambda: b.gen != gen
            if held[slot] != riter:
                raise Violation("team %d reads tile %s from buffer %d, wants tile %d" % (team, held[slot], slot, riter))
            if issued[team][wg] != v or issued[team][1 - wg] != (v + 1 if wg else v):
                raise Violation("team %d warpgroup %d issues virtual tile %d out of turn %s" % (team, wg, v, issued[team]))
            issued[team][wg] += 1
            computed[(riter, cls, wg)] = computed.get((riter, cls, wg), 0) + 1
            if wg == 0 or v + 1 < nv or not skip_last_arrive:
                bar(team, wg).arrive()
            yield lambda: True   # the MMAs complete
            if cls == ncls - 1:
                readers[slot] -= 1
                empty[slot].arrive()
            yield lambda: True   # epilogue

    rng = random.Random(seed)
    actors = [producer()] + [warpgroup(t, g) for t in range(teams) for g in range(2)]
    waits = [next(a, None) for a in actors]
    while any(w is not None for w in waits):
        ready = [i for i, w in enumerate(waits) if w is not None and w()]
        if not ready:
            raise Violation("deadlock: actors %s wait forever" % [i for i, w in enumerate(waits) if w is not None])
        i = rng.choice(ready)
        waits[i] = next(actors[i], None)
    want = {(r, c, g): 1 for r in range(tiles) for c in range(ncls) for g in range(2)}
    if computed != want:
        raise Violation("computed %s" % sorted(set(want.items()) ^ set(computed.items()))[:4])
    pending = {k: b.count for k, b in bars.items() if b.count}
    if pending:
        raise Violation("named barriers left with pending arrivals: %s" % pending)


CONFIGS = [(tiles, ncls, depth, teams) for tiles in range(10) for ncls in (1, 2, 4) for depth in range(2, 9) for teams in (1, 2)]
SEEDS = range(6)


def test_schedule_is_sound():
    for tiles, ncls, depth, teams in CONFIGS:
        for seed in SEEDS:
            simulate(tiles, ncls, depth, teams, seed)


def _failures(**fault):
    bad = set()
    for cfg in CONFIGS:
        for seed in SEEDS:
            try:
                simulate(*cfg, seed, **fault)
            except Violation:
                bad.add(cfg)
    return bad


def test_unskipped_last_arrive_is_caught():
    # warpgroup 1 arriving after its team's last virtual tile leaves that team's barrier half-arrived: every run in which a
    # team has a tile, for one team and for two
    bad = _failures(skip_last_arrive=False)
    assert bad == {c for c in CONFIGS if c[0] >= 1}


def test_shared_barrier_ids_are_caught():
    # two teams on one pair of barriers complete each other's generations. Only runs in which both teams have a tile can
    # fail (one team has nothing to share); with a tile or two per team some interleavings happen to pair up, from four
    # tiles per CTA on every configuration is caught
    bad = _failures(shared_ids=True)
    assert bad <= {c for c in CONFIGS if c[3] == 2 and c[0] >= 2}
    assert bad >= {c for c in CONFIGS if c[3] == 2 and c[0] >= 4}


@pytest.mark.parametrize("teams", [1, 2])
def test_ring_needs_no_buffer_beyond_one_per_team(teams):
    # the kernel's planner asks for four buffers before it runs two teams (to load ahead); the protocol itself is sound at two
    for seed in range(50):
        simulate(9, 4, 2, teams, seed)
