"""Constructed scenes for the object-stacking rules (ObjectStackingComponent): put-downs and pick-ups at the edges of the step kernel's
dense voxel grid and at the boundaries of the scenarios' placement rules.

A scene is one script per env: a generator that warps agents (the oracle's orc_scen_warp; on the GPU the engine then gets the twelve
floats the oracle holds) and yields the action masks of the next tick, {agent: mask}.  All envs of a run advance in lockstep, one tick
per yield.  After each tick the script reads the oracle's record and asserts its reach clause: that the tick did what the family is
built for (an object landed in the voxel it names, outside the grid or in it, a put-down or pick-up was refused, a stack has the heights
it claims).  The same scripts run on the oracle alone (test_stacking_edges_cpu.py) and, tick by tick against the oracle, through the
CUDA step kernel (test_stacking_edges_gpu.py).

The geometry: an agent's object transform is its position + (0, 0.05, 0); the pick point is that, through the camera (0.41 up) and the
pick-up offset (0.44 down, 1 forward), so with a level head it lies 1 ahead of the agent and 0.02 above it.  A carried object hangs
0.3 below the pick point, and a put-down starts in the voxel its translation floors to.  An agent standing on a floor at height h is at
y = h + 0.855; one warped into the air falls about 0.06 in its first tick."""
import ctypes as C
import math

import numpy as np

INTERACT = 1 << 8
AG = 26            # floats per agent in the state dump
DIRS = ((1, 0), (-1, 0), (0, 1), (0, -1))
VOID_Y = -30       # component_object_stacking.hpp: a put-down sinks no lower
AIR = 0.78         # warp height above a voxel's floor at which a carried object starts in that voxel, after one tick's fall
MARGIN = {"collect": 16, "obstacles": 1}  # grid cells beyond the level's horizontal extent (levelgen.cpp)
PARAMS = {"episodeLengthSec": 600.0}      # no episode ends inside a scene


def family(scenario):
    n = scenario.lower()
    if n.startswith("obstacles"):
        return "obstacles"
    return {"towerbuilding": "tower"}.get(n, n)


def yaw_towards(dx, dz):
    """yaw about +Y whose forward vector points along (dx, dz)"""
    return math.atan2(-dx, -dz)


def vox(p):
    return tuple(int(math.floor(float(c))) for c in p)


class OracleRun:
    """the oracle alone, with the interface the scripts use (test_events_gpu.Run adds the engine beside it)"""

    def __init__(self, scenario, E, A, seed, params=None):
        import orc

        self.scenario, self.E, self.A = scenario, E, A
        self.O = orc.lib()
        self.O.orc_scen_warp.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
        self.o = orc.Oracle(scenario, E, A, params=params, render=False, threads=4)
        for e in range(E):
            self.o.seed_env(e, seed + 7919 * e)
        self.o.reset()
        self.states = [self.o.state(e) for e in range(E)]

    def warp(self, e, a, x, y, z, yaw):
        self.O.orc_scen_warp(self.o.h_, e, a, float(x), float(y), float(z), float(yaw))
        self.states[e] = self.o.state(e)

    def step(self, acts, tag):
        self.o.step(acts)
        self.states = [self.o.state(e) for e in range(self.E)]
        return self.o.dones()

    def close(self):
        self.o.close()


class Ctx:
    """what a script sees of env e: the oracle's record and the product's grid box for the env's level"""

    def __init__(self, run, e, seed, params):
        from megaverse_b200 import capi

        self.run, self.e, self.A = run, e, run.A
        self.fam = family(run.scenario)
        self.org, self.dim = capi.grid_box(run.scenario, run.A, seed + 7919 * e, 0, params)
        self.top = int(self.org[1] + self.dim[1])  # first row above the grid
        self.log = []  # (what, detail) of every reach clause met

    # ---- the oracle's record
    def state(self):
        return self.run.states[self.e]

    def agent(self, a):
        return self.state()[8 + AG * a: 8 + AG * (a + 1)]

    def carrying(self, a):
        return int(self.agent(a)[22])

    def objects(self):
        st = self.state()
        n = int(st[5])
        return st[8 + AG * self.A: 8 + AG * self.A + 9 * n].reshape(n, 9)

    def obj_voxel(self, oi):
        return vox(self.objects()[oi][:3])

    def resting(self):
        return [i for i, o in enumerate(self.objects()) if o[6] < 0]

    def occupied(self):
        """voxels holding a solid or an object"""
        v = self.run.o.voxels(self.e)
        return {tuple(int(c) for c in r[:3]) for r in v if r[3] & 5}

    def column_top(self, x, z, occ=None):
        occ = self.occupied() if occ is None else occ
        ys = [y for (vx, y, vz) in occ if vx == x and vz == z]
        return max(ys) if ys else None

    def in_grid(self, v):
        return all(self.org[k] <= v[k] < self.org[k] + self.dim[k] for k in range(3))

    def level_box(self):
        """the level's horizontal extent [lo, hi) in x and z: the grid less its margin"""
        m = MARGIN.get(self.fam, 0)
        return (int(self.org[0]) + m, int(self.org[0] + self.dim[0]) - m), (int(self.org[2]) + m, int(self.org[2] + self.dim[2]) - m)

    def note(self, what, detail):
        self.log.append((what, detail))

    def sides(self, v, a, occ):
        """the directions (dx, dz) from which agent a can stand one voxel back from v, in a free cell with no other agent near, the
        ones with the fewest objects around the cell first (an object's collision box is 1.15 voxels wide and may push the agent
        aside before it interacts)"""
        objs = {tuple(int(c) for c in r[:3]) for r in self.run.o.voxels(self.e) if r[3] & 4}
        others = [self.agent(j)[:3] for j in range(self.A) if j != a]
        out = []
        for dx, dz in DIRS:
            sx, sz = v[0] - dx, v[2] - dz
            if (sx, v[1], sz) in occ or (sx, v[1] + 1, sz) in occ:
                continue
            if any(abs(p[0] - sx - 0.5) < 1.6 and abs(p[2] - sz - 0.5) < 1.6 and abs(p[1] - v[1]) < 3 for p in others):
                continue
            near = [(sx + i, v[1] + h, sz + k) for i in (-1, 0, 1) for k in (-1, 0, 1) for h in (0, 1)]
            out.append((sum(c in objs and (c[0], c[2]) != (v[0], v[2]) for c in near), (dx, dz)))
        return [d for _, d in sorted(out)]

    # ---- moves: each yields the masks of one tick and asserts its outcome after it
    def pick(self, a, oi):
        """stand facing object oi, one voxel from it, and take it; from the next side when the agent was pushed off its aim"""
        t = self.objects()[oi][:3]
        v = vox(t)
        for d in self.sides(v, a, self.occupied()):
            self.run.warp(self.e, a, t[0] - d[0], v[1] + 0.855, t[2] - d[1], yaw_towards(*d))
            yield {a: INTERACT}
            if self.carrying(a) == oi:
                return True
            assert self.carrying(a) < 0, "env %d agent %d: picked %d, meant %d at %s" % (self.e, a, self.carrying(a), oi, v)
        return False

    def pick_free(self, a, avoid=()):
        """take a resting object on the level (not in the void) that no script has claimed (not in `avoid`), with nothing on it"""
        occ = self.occupied()
        for oi in self.resting():
            v = self.obj_voxel(oi)
            if oi in avoid or v[1] < 0 or not self.in_grid(v) or (v[0], v[1] + 1, v[2]) in occ:
                continue
            if (yield from self.pick(a, oi)):
                return oi
            occ = self.occupied()
        raise AssertionError("env %d agent %d: no object left to pick up" % (self.e, a))

    def put(self, a, x, y, z, d=None):
        """put agent a's object down from voxel (x, y, z), standing one voxel back along d (any free side when None); returns its
        landing voxel, or None when the put-down was refused"""
        oi = self.carrying(a)
        assert oi >= 0, "env %d agent %d carries nothing" % (self.e, a)
        if d is None:
            d = self.sides((x, y, z), a, self.occupied())[0]
        dx, dz = d
        self.run.warp(self.e, a, x + 0.5 - dx, y + AIR, z + 0.5 - dz, yaw_towards(dx, dz))
        yield {a: INTERACT}
        if self.carrying(a) == oi:
            return None
        assert self.carrying(a) < 0 and self.objects()[oi][6] < 0
        return self.obj_voxel(oi)

    def put_on_column(self, a, x, z, above=1):
        """put down `above` voxels over the column's top (solid or object), from a free side"""
        occ = self.occupied()
        tops = [self.column_top(x, z, occ)] + [self.column_top(x - dx, z - dz, occ) for dx, dz in DIRS]
        y = max(t for t in tops if t is not None) + above
        return (yield from self.put(a, x, y, z))

    def wait(self, n=1):
        for _ in range(n):
            yield {}


def parallel(*gens):
    """run scripts of different agents of one env side by side: each tick merges their masks; returns their results"""
    gens = list(gens)
    out = [None] * len(gens)
    live = list(range(len(gens)))
    while live:
        masks = {}
        for i in list(live):
            try:
                masks.update(next(gens[i]))
            except StopIteration as stop:
                out[i] = stop.value
                live.remove(i)
        if live:
            yield masks
    return out


# ------------------------------------------------------------------------------------------------ families
def void_column(ctx, face, dists):
    """a carrying agent puts down beyond face `face` (0..3: +x, -x, +z, -z) at each distance in `dists` from the level's last column
    (0), through the margin, to past the grid; from above the level, so it sinks down the column.  Agents share out the distances."""
    (x0, x1), (z0, z1) = ctx.level_box()
    m = MARGIN[ctx.fam]
    dx, dz = DIRS[face]
    y = ctx.top - 1

    def column(d, a):  # agents work side by side, three columns apart
        if dx:
            return (x1 - 1 + d if dx > 0 else x0 - d), (z0 + z1) // 2 + 3 * a
        return (x0 + x1) // 2 + 3 * a, (z1 - 1 + d if dz > 0 else z0 - d)

    claimed = set()

    def agent(a, mine):
        for d in mine:
            claimed.add((yield from ctx.pick_free(a, avoid=claimed)))
            x, z = column(d, a)
            land = yield from ctx.put(a, x, y, z, (dx, dz))
            assert land is not None and land[0] == x and land[2] == z, "env %d: face %d d=%d landed at %s" % (ctx.e, face, d, land)
            if d > m:  # reach: beyond the grid's side, sunk to the bottom of the void
                assert land[1] == VOID_Y and not ctx.in_grid(land), "env %d: d=%d landed at %s (grid %s %s)" % (ctx.e, d, land, ctx.org, ctx.dim)
                ctx.note("void_outside", land)
            else:
                assert ctx.in_grid(land), "env %d: d=%d landed at %s outside the grid" % (ctx.e, d, land)
                ctx.note("column_inside", (d, land))

    yield from parallel(*[agent(a, dists[a::ctx.A]) for a in range(ctx.A)])


def void_stack(ctx, k, face=0):
    """k put-downs into one column beyond the grid, then one into the column beside it: heights -30, -29, ... and -30 again.  With
    A >= 2 the agents put down in the same tick, in agent order."""
    (x0, x1), (z0, z1) = ctx.level_box()
    m = MARGIN[ctx.fam]
    dx, dz = DIRS[face]
    d = m + 3
    x, z = ((x1 - 1 + d if dx > 0 else x0 - d), (z0 + z1) // 2) if dx else ((x0 + x1) // 2, (z1 - 1 + d if dz > 0 else z0 - d))
    side = (x, z + 1) if dx else (x + 1, z)
    claimed = set()
    heights = []
    puts = [(x, z)] * k + [side]
    for i in range(0, len(puts), ctx.A):
        batch = puts[i:i + ctx.A]
        for a in range(len(batch)):
            claimed.add((yield from ctx.pick_free(a, avoid=claimed)))
        # the agents of a batch stand on opposite sides of the column
        lands = yield from parallel(*[ctx.put(a, c[0], ctx.top - 1, c[1], (dx, dz) if a % 2 == 0 else (-dx, -dz)) for a, c in enumerate(batch)])
        heights += lands
    want = [(x, VOID_Y + i, z) for i in range(k)] + [(side[0], VOID_Y, side[1])]
    assert heights == want, "env %d: stack %s, want %s" % (ctx.e, heights, want)
    assert not any(ctx.in_grid(v) for v in heights)
    ctx.note("void_stack", [v[1] for v in heights])
    return (x, z), (dx, dz)


def void_pickup(ctx):
    """Collect: a void stack whose top reaches y = -20, picked from an agent warped to y = -19.5 beside it (the fall reset is at -20);
    then, two objects higher, the same reach finds an object above every voxel it tries and takes nothing"""
    (x, z), (dx, dz) = yield from void_stack(ctx, 11)
    assert ctx.column_top(x, z) == -20

    def reach(a):
        ctx.run.warp(ctx.e, a, x + 0.5 - dx, -19.5, z + 0.5 - dz, yaw_towards(dx, dz))
        yield {a: INTERACT}

    top = next(i for i in ctx.resting() if ctx.obj_voxel(i) == (x, -20, z))
    yield from reach(0)
    assert ctx.carrying(0) == top, "env %d: the void stack's top was not picked up (%d)" % (ctx.e, ctx.carrying(0))
    ctx.note("void_pickup", top)
    yield from ctx.wait(2)  # the agent falls below -20 and is reset, still carrying
    for y in (-20, -19, -18):
        if ctx.carrying(0) < 0:
            yield from ctx.pick_free(0)
        land = yield from ctx.put(0, x, ctx.top - 1, z, (dx, dz))
        assert land == (x, y, z), "env %d: landed at %s, want y %d" % (ctx.e, land, y)
    a = 1 if ctx.A > 1 else 0
    yield from reach(a)
    assert ctx.carrying(a) < 0, "env %d: picked %d under two objects" % (ctx.e, ctx.carrying(a))
    assert ctx.column_top(x, z) == -18
    ctx.note("void_pickup_blocked", (x, z))


def above_top(ctx, column, tower=None):
    """a put-down that starts above the grid's top face and sinks into it.  With `tower` objects to spare, a column is built on
    `column` to the grid's top row: a pick-up there (the voxel above is outside the grid), and one put-down more, which lands above
    the grid; it is then picked up from there."""
    x, z = column
    a = 0
    yield from ctx.pick_free(a)
    land = yield from ctx.put(a, x, ctx.top + 2, z)
    assert land is not None and ctx.in_grid(land) and land[1] < ctx.top, "env %d: from above the top landed at %s" % (ctx.e, land)
    ctx.note("from_above", land)
    if not tower:
        return
    while ctx.column_top(x, z) < ctx.top - 1:
        yield from ctx.pick_free(a, avoid={i for i in ctx.resting() if ctx.obj_voxel(i)[0] == x and ctx.obj_voxel(i)[2] == z})
        land = yield from ctx.put_on_column(a, x, z)
        assert land is not None and land[0] == x and land[2] == z
    assert ctx.column_top(x, z) == ctx.top - 1
    row = next(i for i in ctx.resting() if ctx.obj_voxel(i) == (x, ctx.top - 1, z))
    assert (yield from ctx.pick(a, row))  # the top row: the voxel above is outside the grid
    ctx.note("top_row_pickup", row)
    land = yield from ctx.put_on_column(a, x, z)
    assert land == (x, ctx.top - 1, z)
    yield from ctx.pick_free(a, avoid={row})
    land = yield from ctx.put_on_column(a, x, z)
    assert land == (x, ctx.top, z) and not ctx.in_grid(land), "env %d: past the head-room landed at %s" % (ctx.e, land)
    ctx.note("past_headroom", land)
    over = next(i for i in ctx.resting() if ctx.obj_voxel(i) == land)
    assert (yield from ctx.pick(a, over))
    ctx.note("past_headroom_pickup", over)


def zone_edges(ctx):
    """TowerBuilding: put-downs at x and z = bz_min - 1, bz_min, bz_max - 1, bz_max (the other coordinate mid-zone): refused outside,
    accepted inside, the building reward and highest tower following; then the accepted ones picked up again from the edge cells"""
    L = ctx.run.o.level(ctx.e)
    mn, mx = L[3:6], L[6:9]
    mid = ((mn[0] + mx[0]) // 2, (mn[2] + mx[2]) // 2)
    targets = []
    for axis in (0, 2):
        for c in (mn[axis] - 1, mn[axis], mx[axis] - 1, mx[axis]):
            targets.append((c, mid[1]) if axis == 0 else (mid[0], c))
    placed = []

    def zone_objects():
        return [i for i in ctx.resting() if mn[0] <= ctx.obj_voxel(i)[0] < mx[0] and mn[2] <= ctx.obj_voxel(i)[2] < mx[2]]

    for x, z in targets:
        inside = mn[0] <= x < mx[0] and mn[2] <= z < mx[2]
        if ctx.carrying(0) < 0:  # from outside the zone: a pick-up in the zone drops its voxel from the set without paying
            yield from ctx.pick_free(0, avoid=placed + zone_objects())
        oi = ctx.carrying(0)
        st = ctx.state().copy()
        occ = ctx.occupied()
        top = ctx.column_top(x, z, occ)
        assert top is not None and (x, top + 1, z) not in occ
        land = yield from ctx.put_on_column(0, x, z)
        if inside:
            assert land is not None and (land[0], land[2]) == (x, z), "env %d: zone cell %s refused" % (ctx.e, (x, z))
            assert ctx.state()[4] > st[4] and ctx.state()[3] >= land[1] - mn[1] + 1, "env %d: tower reward / height did not follow" % ctx.e
            placed.append(oi)
            ctx.note("zone_accepted", (x, z))
        else:
            assert land is None, "env %d: cell %s outside the zone accepted (landed %s)" % (ctx.e, (x, z), land)
            ctx.note("zone_refused", (x, z))
    for oi in placed:  # pick-ups from the edge cells: the building zone set loses them, which the next put-down's reward shows
        if ctx.carrying(0) >= 0:
            land = yield from ctx.put_on_column(0, mid[0], mid[1])
            assert land is not None
        assert (yield from ctx.pick(0, oi))
        ctx.note("zone_pickup", oi)
    land = yield from ctx.put_on_column(0, mid[0], mid[1])
    assert land is not None


def pedestal_edges(ctx):
    """Rearrange: put-downs at |dx| or |dz| of 2 from the work centre are accepted, 3 refused"""
    c = ctx.run.o.arrangement(ctx.e)[-3:]  # rightCenter
    targets = [(c[0] + s * k, c[2]) for k in (2, 3) for s in (1, -1)] + [(c[0], c[2] + s * k) for k in (2, 3) for s in (1, -1)]
    targets += [(c[0] + 2, c[2] + 2), (c[0] - 2, c[2] + 3)]
    for x, z in targets:
        ok = abs(x - c[0]) <= 2 and abs(z - c[2]) <= 2
        if ctx.carrying(0) < 0:
            yield from ctx.pick_free(0)
        land = yield from ctx.put_on_column(0, x, z)
        if ok:
            assert land is not None and (land[0], land[2]) == (x, z), "env %d: pedestal cell %s refused" % (ctx.e, (x, z))
            ctx.note("pedestal_accepted", (x - c[0], z - c[2]))
        else:
            assert land is None, "env %d: cell %s off the pedestal accepted" % (ctx.e, (x, z))
            ctx.note("pedestal_refused", (x - c[0], z - c[2]))


def agent_in_target(ctx, cells):
    """agent 1 stands on a cell; agent 0's put-down into agent 1's voxel is refused, one voxel to the side accepted"""
    assert ctx.A >= 2
    for x, z in cells:
        if ctx.carrying(0) < 0:
            yield from ctx.pick_free(0)
        top = ctx.column_top(x, z)
        ctx.run.warp(ctx.e, 1, x + 0.5, top + 1 + 0.855, z + 0.5, 0.0)
        yield from ctx.wait(3)
        v1 = vox(ctx.agent(1)[:3] + np.float32([0, 0.05, 0]))
        assert (v1[0], v1[2]) == (x, z)
        occ = ctx.occupied()
        d = next((dx, dz) for dx, dz in DIRS if all((x - dx, v1[1] + h, z - dz) not in occ for h in (0, 1))
                 and all((x + dz, v1[1] + h, z + dx) not in occ for h in (0, 1)) and ctx.column_top(x + dz, z + dx, occ) == top)
        land = yield from ctx.put(0, v1[0], v1[1], v1[2], d)
        assert land is None, "env %d: put-down into agent 1's voxel %s accepted" % (ctx.e, v1)
        ctx.note("agent_refused", v1)
        land = yield from ctx.put(0, x + d[1], v1[1], z + d[0], d)
        assert land is not None and (land[0], land[2]) == (x + d[1], z + d[0]), "env %d: beside agent 1 refused (%s)" % (ctx.e, land)
        ctx.note("agent_beside_accepted", land)


def pickup_height(ctx, column):
    """a stack of 1, 2, 3 objects on one column, each picked at its bottom voxel: the object itself; the one above (the bottom is
    covered, so the rule tries one voxel higher); nothing (both tried voxels covered)"""
    x, z = column
    base = ctx.column_top(x, z) + 1
    stack = []
    for n in (1, 2, 3):
        while len(stack) < n:
            if ctx.carrying(0) < 0:
                yield from ctx.pick_free(0, avoid=stack)
            oi = ctx.carrying(0)
            land = yield from ctx.put_on_column(0, x, z)
            assert land == (x, base + len(stack), z), "env %d: stack landed at %s" % (ctx.e, land)
            stack.append(oi)
        occ = ctx.occupied()
        dx, dz = next((dx, dz) for dx, dz in DIRS if (x - dx, base, z - dz) not in occ and (x - dx, base + 1, z - dz) not in occ
                      and ctx.column_top(x - dx, z - dz, occ) == base - 1)
        ctx.run.warp(ctx.e, 0, x + 0.5 - dx, base + 0.855, z + 0.5 - dz, yaw_towards(dx, dz))
        yield {0: INTERACT}
        got = ctx.carrying(0)
        if n == 1:
            assert got == stack[0], "env %d: the single object was not picked (%d)" % (ctx.e, got)
        elif n == 2:
            assert got == stack[1], "env %d: with one above, picked %d, want the upper %d" % (ctx.e, got, stack[1])
        else:
            assert got < 0, "env %d: picked %d from under two objects" % (ctx.e, got)
        ctx.note("pickup_height_%d" % n, got)
        if got >= 0:  # back on top
            stack.remove(got)
            land = yield from ctx.put_on_column(0, x, z)
            assert land == (x, base + len(stack), z)
            stack.append(got)


# ------------------------------------------------------------------------------------------------ scenes
def level_objects(scenario, A, seed, params):
    from megaverse_b200 import capi

    return int(capi.generate_level(scenario, A, seed, 0, params)[2])


def spread(ctx, i):
    """a column of the level away from objects and walls for scene i: the i-th of the level's free floor cells in scan order"""
    occ = ctx.occupied()
    (x0, x1), (z0, z1) = ctx.level_box() if ctx.fam in MARGIN else ((int(ctx.org[0]) + 1, int(ctx.org[0] + ctx.dim[0]) - 1),
                                                                    (int(ctx.org[2]) + 1, int(ctx.org[2] + ctx.dim[2]) - 1))
    objs = {ctx.obj_voxel(o)[::2] for o in ctx.resting()}
    cells = []
    for x in range(x0 + 1, x1 - 1):
        for z in range(z0 + 1, z1 - 1):
            t = ctx.column_top(x, z, occ)
            if t is None or (x, z) in objs:
                continue
            nb = [ctx.column_top(x + dx, z + dz, occ) for dx, dz in DIRS]
            if all(n == t for n in nb) and not any((x + dx, z + dz) in objs for dx, dz in DIRS):
                cells.append((x, z))
    assert cells, "env %d: no flat free cell" % ctx.e
    return cells[(i * 7919) % len(cells)]


# name -> (scenario, A, E, seed, script(ctx) -> generator, objects each env needs)
def _void_columns(ctx):
    m = MARGIN[ctx.fam]
    return void_column(ctx, ctx.e % 4, sorted({0, 1, m, m + 1, 30}))


def _void_stack(ctx):
    return void_stack(ctx, 10 if ctx.fam == "collect" else 4, face=ctx.e % 4)


def zone_cell(ctx, i):
    """TowerBuilding: the i-th free floor cell of the building zone (put-downs count only there)"""
    L = ctx.run.o.level(ctx.e)
    occ = ctx.occupied()
    cells = [(x, z) for x in range(L[3], L[6]) for z in range(L[5], L[8]) if ctx.column_top(x, z, occ) == L[4] - 1]
    return cells[(i * 7919) % len(cells)]


def _above_top(ctx):
    if ctx.fam == "tower":
        return above_top(ctx, zone_cell(ctx, ctx.e), tower=ctx.e == 0)
    return above_top(ctx, spread(ctx, ctx.e))


def work_centre(ctx):
    """Rearrange: the (x, z) of the work centre (rightCenter), where put-downs are allowed"""
    c = ctx.run.o.arrangement(ctx.e)[-3:]
    return int(c[0]), int(c[2])


def _zone_and_height(ctx):
    return zone_edges(ctx) if ctx.e % 2 == 0 else pickup_height(ctx, zone_cell(ctx, ctx.e))


def _agents(ctx):
    return agent_in_target(ctx, [spread(ctx, ctx.e + k) for k in range(2)])


SCENES = {
    "void_columns_obstacles": ("ObstaclesHard", 1, 4, 11, _void_columns, 6),
    "void_columns_obstacles_a2": ("ObstaclesMedium", 2, 4, 12, _void_columns, 6),
    "void_columns_collect": ("Collect", 2, 4, 13, _void_columns, 5),
    "void_stack_obstacles": ("ObstaclesWalls", 2, 4, 14, _void_stack, 5),
    "void_stack_collect": ("Collect", 1, 4, 15, _void_stack, 11),
    "void_pickup_collect": ("Collect", 2, 2, 16, void_pickup, 16),
    "above_top_tower": ("TowerBuilding", 1, 2, 17, _above_top, 30),
    "above_top_collect": ("Collect", 1, 2, 18, _above_top, 1),
    "above_top_obstacles": ("ObstaclesEasy", 1, 2, 19, _above_top, 1),
    "above_top_rearrange": ("Rearrange", 1, 2, 20, lambda ctx: above_top(ctx, work_centre(ctx)), 1),
    "zone_edges_and_pickup_height_tower": ("TowerBuilding", 1, 4, 21, _zone_and_height, 6),
    "pedestal_edges_rearrange": ("Rearrange", 1, 2, 22, pedestal_edges, 3),
    "pickup_height_collect": ("Collect", 2, 2, 23, lambda ctx: pickup_height(ctx, spread(ctx, ctx.e)), 4),
    "agent_in_target_collect": ("Collect", 2, 2, 24, _agents, 2),
    "agent_in_target_obstacles": ("ObstaclesHard", 3, 2, 25, _agents, 2),
}


def scene_seed(name, A, E):
    """the first seed from the scene's own on whose E levels every env has the objects its script needs"""
    scenario, _, _, seed, _, need = SCENES[name]
    for s in range(seed, seed + 400 * 997, 997):
        if all(level_objects(scenario, A, s + 7919 * e, PARAMS) >= need for e in range(E)):
            return s
    raise AssertionError("%s: no seed with %d objects per level" % (name, need))


def play(run, scripts, check=None):
    """advance every env's script one tick at a time; check(run, tag) after every tick (the GPU test's comparisons)"""
    gens = list(scripts)
    live = [True] * len(gens)
    t = 0
    while True:
        acts = np.zeros(run.E * run.A, dtype=np.int32)
        for e, g in enumerate(gens):
            if not live[e]:
                continue
            try:
                for a, m in next(g).items():
                    acts[e * run.A + a] = m
            except StopIteration:
                live[e] = False
        if not any(live):
            return t
        tag = "%s t=%d" % (run.scenario, t)
        d = run.step(acts, tag)
        assert not np.any(d), "%s: an episode ended inside the scene" % tag
        if check:
            check(run, tag)
        t += 1


def run_scene(name, make_run, check=None):
    """play scene `name` on make_run(scenario, E, A, seed, params), closed at the end; returns (ctxs, ticks)"""
    scenario, A, E, _, script, _ = SCENES[name]
    seed = scene_seed(name, A, E)
    run = make_run(scenario, E, A, seed, PARAMS)
    try:
        ctxs = [Ctx(run, e, seed, PARAMS) for e in range(E)]
        if check:
            check(run, "%s reset" % name)
        return ctxs, play(run, [script(c) for c in ctxs], check)
    finally:
        run.close()
