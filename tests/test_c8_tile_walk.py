"""Which tile each conv_c8_kernel CTA, team and iteration computes, as a CPU model of the launch plan and the tile walks.

The model is written from DESIGN.md 5.1, not from the kernel's code. The host launches grid = min(tiles, SMs) CTAs
(streamed weights: 2-CTA clusters, grid = 2 min(ceil(tiles / 2), clusters that fit)) and runs two teams of consumer
warpgroups when the layer's plan allows them and its CTAs run at least two tiles. Tiles are 16 rows x 8 columns, numbered
tile = (img tiles_y + ty) tiles_x + tx. CTA b's producer loads tiles b, b + grid, ... into halo ring slot (its iteration
mod a_bufs); team t of CTA b runs that CTA's iterations riter = t, t + TEAMS, ... (each over all fused classes). Neither
divides per tile: each steps (tx, ty, img) in mixed radix by `step` (the grid) or `cstep` (TEAMS x the grid), decomposed
once on the host, with one carry from x into y and one from y into img. A cluster's CTAs run for as long as the pair's
rank-0 tile exists; with an odd tile count the last pair's rank 1 is a phantom that loads and computes nothing.

Checked over a broad grid of batches, tile grids, SM counts (132 and 114, 78 and 7 as well) and launch kinds: every tile
(and class) is computed exactly once, by the CTA whose producer loaded it into ring slot riter mod a_bufs; the producer's
and each team's coordinates equal the closed form of their tile number; no coordinate leaves its range after its one
carry. The model is shown to fail when the x -> y carry is dropped, when the teams step by the grid instead of TEAMS x the
grid, and when team 1 starts at blockIdx.x + 1, on the geometries where those faults change the walk.
"""
import pytest


class Violation(Exception):
    pass


SMS = (132, 114, 78, 7)
KINDS = ("one", "teams", "cluster")   # resident one team, resident with a two-team form, streamed (clustered)
FAULTS = ("no_x_carry", "cstep_is_grid", "team1_at_plus1")


def plan(kind, N, tiles_x, tiles_y, sms):
    """the host's launch: grid, teams, cluster and the two mixed-radix steps."""
    per = tiles_x * tiles_y
    total = N * per
    grid = min(total, sms)
    cluster = 2 if kind == "cluster" else 1
    teams = 2 if kind == "teams" and total > grid else 1
    if cluster == 2:
        grid = 2 * min((total + 1) // 2, sms // 2)   # one CTA per SM: sms // 2 clusters fit
    decomp = lambda s: (s % tiles_x, s // tiles_x % tiles_y, s // per)
    return dict(N=N, tiles_x=tiles_x, tiles_y=tiles_y, total=total, grid=grid, teams=teams, cluster=cluster, sms=sms,
                step=decomp(grid), cstep=decomp(teams * grid))


def decode(tile, tiles_x, tiles_y):
    return tile % tiles_x, tile // tiles_x % tiles_y, tile // (tiles_x * tiles_y)


def walk(p, a_bufs=4, ncls=1, fault=None, events=None):
    """run every CTA's producer and teams; returns {(img, ty, tx, cls): times computed}. Raises Violation."""
    tx_n, ty_n, total, grid, teams = p["tiles_x"], p["tiles_y"], p["total"], p["grid"], p["teams"]
    clustered = p["cluster"] > 1

    def advance(c, step, tile):
        """one mixed-radix step to `tile` (events of steps to real tiles only: a phantom's coordinates are never used)"""
        x, y, img = c
        ev = set()
        x += step[0]
        if x >= tx_n:
            x -= tx_n
            if fault != "no_x_carry":
                y += 1
            ev.add("x_carry")
        y += step[1]
        if y >= ty_n:
            y -= ty_n
            img += 1
            if "x_carry" in ev:
                ev.add("xyimg_carry")   # x carried into y and y into img on the same step
        img += step[2]
        if not (0 <= x < tx_n and 0 <= y < ty_n):
            raise Violation("coordinate (%d, %d) out of range after one carry" % (x, y))
        if events is not None and tile < total:
            events.update(ev)
        return x, y, img

    computed = {}
    iters = {}
    for b in range(grid):
        rank = b % 2 if clustered else 0
        # producer: one halo per tile into ring slot (iteration mod a_bufs); a phantom loads nothing
        loads = []
        c = decode(b, tx_n, ty_n)
        tile, it = b, 0
        while tile - rank < total:
            if tile != b:
                c = advance(c, p["step"], tile)
            if tile < total:
                if c != decode(tile, tx_n, ty_n):
                    raise Violation("producer of CTA %d at tile %d holds %s" % (b, tile, c))
                loads.append((it % a_bufs, c))
            elif not (clustered and rank == 1 and tile == total):
                raise Violation("CTA %d loads past the last tile (%d)" % (b, tile))
            else:
                loads.append(None)
            tile += grid
            it += 1
        iters[b] = it
        # teams: team t runs the CTA's iterations t, t + teams, ... and every class of each
        first = b - rank
        my_tiles = (total - first + grid - 1) // grid if first < total else 0
        if my_tiles != it:
            raise Violation("CTA %d: consumers count %d tiles, the producer %d" % (b, my_tiles, it))
        for t in range(teams):
            nv = (my_tiles - t + teams - 1) // teams * ncls if my_tiles > t else 0
            riter, cls = t, 0
            c = decode(b + (t if fault == "team1_at_plus1" else t * grid), tx_n, ty_n)
            for v in range(nv):
                if v > 0:
                    cls += 1
                    if cls == ncls:
                        cls = 0
                        riter += teams
                        c = advance(c, p["step"] if fault == "cstep_is_grid" else p["cstep"], b + riter * grid)
                tile = b + riter * grid
                if tile >= total:
                    if not (clustered and rank == 1 and loads[riter] is None):
                        raise Violation("CTA %d team %d runs past the last tile" % (b, t))
                    continue
                slot, held = loads[riter]
                if slot != riter % a_bufs or held != c:
                    raise Violation("CTA %d team %d computes %s from slot %d holding %s" % (b, t, c, slot, held))
                if c != decode(tile, tx_n, ty_n):
                    raise Violation("CTA %d team %d at tile %d holds %s" % (b, t, tile, c))
                key = (c[2], c[1], c[0], cls)
                computed[key] = computed.get(key, 0) + 1
    if clustered:
        for b in range(0, grid, 2):
            if iters[b] != iters[b + 1]:
                raise Violation("cluster %d: ranks run %d and %d tiles" % (b // 2, iters[b], iters[b + 1]))
    want = {(img, y, x, k): 1 for img in range(p["N"]) for y in range(ty_n) for x in range(tx_n) for k in range(ncls)}
    if computed != want:
        diff = sorted(set(want.items()) ^ set(computed.items()))[:4]
        raise Violation("tiles computed other than once: %s" % diff)
    return computed


def geometries(p, events):
    """the named walk geometries a plan and its (sound) walk fall under."""
    per = p["tiles_x"] * p["tiles_y"]
    g = set()
    if p["grid"] > per:
        g.add("step_over_one_image")
    if per == 1 and p["N"] > 2 * p["sms"]:
        g.add("one_tile_images")
    if p["tiles_x"] > p["grid"]:
        g.add("tiles_x_over_step")
    if p["grid"] % per == 0 and p["grid"] >= per:
        g.add("step_multiple_of_image")
    if "xyimg_carry" in events:
        g.add("xyimg_carry")
    if p["cluster"] > 1 and p["total"] % 2:
        g.add("phantom")
    return g


def _configs():
    out = []
    for sms in SMS:
        for kind in KINDS:
            for tiles_x in (1, 2, 3, 5, 8, 12, sms + 5):
                for tiles_y in (1, 2, 3, 7, 11):
                    for N in (1, 2, 3, 7, 2 * sms + 3):
                        if N * tiles_x * tiles_y <= 6000:
                            out.append((sms, kind, N, tiles_x, tiles_y))
    return out


CONFIGS = _configs()


def _run(cfg, fault=None, events=None):
    sms, kind, N, tiles_x, tiles_y = cfg
    p = plan(kind, N, tiles_x, tiles_y, sms)
    a_bufs = {"one": 2, "teams": 4, "cluster": 2}[kind]
    walk(p, a_bufs=a_bufs, fault=fault, events=events)
    return p


@pytest.fixture(scope="module")
def sound():
    """{config: (plan, events, geometries)} of the sound walk over every configuration."""
    out = {}
    for cfg in CONFIGS:
        ev = set()
        p = _run(cfg, events=ev)
        out[cfg] = (p, ev, geometries(p, ev))
    return out


def test_every_named_geometry_is_walked(sound):
    # each SM count walks each named geometry with each launch kind it can occur in (phantoms: clusters only)
    named = ("step_over_one_image", "one_tile_images", "tiles_x_over_step", "step_multiple_of_image", "xyimg_carry")
    for sms in SMS:
        for kind in KINDS:
            seen = set().union(*(g for cfg, (p, _, g) in sound.items() if cfg[0] == sms and cfg[1] == kind))
            assert set(named) <= seen, (sms, kind, set(named) - seen)
            if kind == "cluster":
                assert "phantom" in seen, sms
        two = [cfg for cfg, (p, _, _) in sound.items() if cfg[0] == sms and p["teams"] == 2]
        assert two, sms


@pytest.mark.parametrize("ncls", [1, 2, 4])
@pytest.mark.parametrize("a_bufs", [2, 3, 4, 8])
def test_fused_classes_and_ring_depths(ncls, a_bufs):
    # fused classes advance the walk once per tile; the ring slot of a tile does not depend on the team
    for sms in (132, 7):
        for kind in ("one", "teams"):
            for N, tx, ty in ((1, 1, 1), (2 * sms + 3, 1, 1), (3, sms + 5, 2), (5, 3, 7), (2, 12, 11)):
                walk(plan(kind, N, tx, ty, sms), a_bufs=a_bufs, ncls=ncls)


def _caught(cfgs, fault):
    bad = set()
    for cfg in cfgs:
        try:
            _run(cfg, fault=fault)
        except Violation:
            bad.add(cfg)
    return bad


def test_dropped_x_carry_is_caught(sound):
    # caught exactly where the sound walk carries x into y on the way to a real tile: on every x-y-img carry, and on the
    # tiles_x > step grids whose walk wraps a row (one image of 137 x 1 tiles on 132 SMs does not)
    bad = _caught(CONFIGS, "no_x_carry")
    assert bad == {cfg for cfg, (_, ev, _) in sound.items() if "x_carry" in ev}
    for sms in SMS:
        for kind in KINDS:
            of = lambda geo: {cfg for cfg, (_, _, g) in sound.items() if cfg[:2] == (sms, kind) and geo in g}
            assert of("xyimg_carry") and of("xyimg_carry") <= bad, (sms, kind)
            assert of("tiles_x_over_step") & bad, (sms, kind)


def test_teams_stepping_by_the_grid_is_caught(sound):
    # caught wherever a team runs a second tile: two teams and more than two tiles per CTA's first pair of iterations
    bad = _caught(CONFIGS, "cstep_is_grid")
    assert bad == {cfg for cfg, (p, _, _) in sound.items() if p["teams"] == 2 and p["total"] > 2 * p["grid"]}
    for sms in SMS:
        for geo in ("one_tile_images", "step_multiple_of_image", "step_over_one_image"):
            cfgs = {cfg for cfg, (p, _, g) in sound.items() if cfg[0] == sms and p["teams"] == 2 and geo in g}
            assert cfgs & bad, (sms, geo)


def test_team1_starting_one_tile_on_is_caught(sound):
    # team 1 has a tile in every two-team launch (its CTAs run at least two): every one of them fails
    bad = _caught(CONFIGS, "team1_at_plus1")
    assert bad == {cfg for cfg, (p, _, _) in sound.items() if p["teams"] == 2}
    for sms in SMS:
        for geo in ("one_tile_images", "tiles_x_over_step", "step_multiple_of_image", "xyimg_carry"):
            cfgs = {cfg for cfg, (p, _, g) in sound.items() if cfg[0] == sms and p["teams"] == 2 and geo in g}
            assert cfgs and cfgs <= bad, (sms, geo)
