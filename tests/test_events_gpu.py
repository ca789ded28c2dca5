"""Scenario event parity: every reward rule, solved-episode end and fall / lava reset of the step kernel against the oracle, on the GPU.

Random and purposeful walks seldom cross an obstacle course, solve a Boxoban room or walk off a Collect map, so these runs move agents:
each env is warped on its own schedule -- onto exit, lava and reward cells, next to objects, boxes and collectables, below the level --
through the oracle's orc_scen_warp (the character controller's warp), and the twelve floats the oracle then holds go to the engine
through mv_debug_warp_agent.  Every tick the rewards, dones and true objectives are compared bit for bit; right after every warp, every
25 ticks and at every episode end the whole state, the voxels, the frames (byte-exact with fast_shading=0) and the depth as well.

In the coverage runs team spirit is 0 and the reward slots of a scenario are 1, 16, 256, 4096, scaled by 2**a for agent a, so that
each tick's reward decodes into the events that fired; each run asserts that every rule its levels offer fired, and that every solved
rule ended an episode before its timer.  TowerBuilding's building reward (a non-integer multiplier) is 1/256 and is counted from the
state's building-zone reward instead."""
import ctypes as C
import math

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

FWD, INTERACT = 1 << 3, 1 << 8
DT = 1.0 / 15.0
AG = 26  # floats per agent in the state dump

# reward keys in slot order (include/ and levelgen.cpp defaultRewardShaping); slot k of a coverage run is worth 16**k
KEYS = {
    "tower": ["towerPickedUpObject", "towerVisitedBuildingZoneWithObject", "towerBuildingReward"],
    "obstacles": ["obstaclesAgentAtExit", "obstaclesAllAgentsAtExit", "obstaclesExtraReward", "obstaclesAgentCarriedObjectToExit"],
    "collect": ["collectSingleGood", "collectSingleBad", "collectAll", "collectAbyss"],
    "sokoban": ["sokobanBoxOnTarget", "sokobanBoxLeavesTarget", "sokobanAllBoxesOnTarget"],
    "rearrange": ["rearrangeOneMoreObjectCorrectPosition", "rearrangeAllObjectsCorrectPosition"],
    "hexexplore": ["exploreSolved"],
    "hexmemory": ["memoryCollectGood", "memoryCollectBad"],
    "empty": [],
}
# the event each slot stands for in the printed table
EVENTS = {
    "tower": ["picked_up", "visited_zone", "building"],
    "obstacles": ["at_exit", "all_at_exit", "extra", "carried_to_exit"],
    "collect": ["good", "bad", "all_collected", "abyss"],
    "sokoban": ["on_target", "leaves_target", "all_on_target"],
    "rearrange": ["one_more", "all_matched"],
    "hexexplore": ["solved"],
    "hexmemory": ["good", "bad"],
    "empty": [],
}
# rules that end an episode early (doneWithTimer); HexMemory's has no reward of its own
SOLVED = {"obstacles": "all_at_exit", "collect": "all_collected", "sokoban": "all_on_target", "rearrange": "all_matched",
          "hexexplore": "solved", "hexmemory": "all_good"}
FALLS = ("tower", "obstacles", "collect")  # scenarios with FallDetectionComponent


def family(scenario):
    n = scenario.lower()
    if n.startswith("obstacles") or n == "test":
        return "obstacles"
    return {"towerbuilding": "tower"}.get(n, n)


def yaw_towards(dx, dz):
    """yaw about +Y whose forward vector (basis row 2, z negated) points along (dx, dz)"""
    return math.atan2(-dx, -dz)


class Run:
    """one CUDA engine and one oracle on the same env seeds; the oracle renders only at checkpoints"""

    def __init__(self, scenario, E, A, seed, params=None, fast_shading=False, coverage=True, team_spirit=None):
        import orc
        from megaverse_b200 import capi

        self.scenario, self.fam, self.E, self.A = scenario, family(scenario), E, A
        self.fast = fast_shading
        self.O = orc.lib()
        self.O.orc_scen_warp.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
        self.o = orc.Oracle(scenario, E, A, params=params, render=False, depth=True, threads=4)
        self.g = capi.Engine(scenario, E, A, num_threads=4, params=params, depth=True)
        self.g.set_option("fast_shading", 1 if fast_shading else 0)
        for e in range(E):
            self.o.seed_env(e, seed + 7919 * e)
            self.g.seed_env(e, seed + 7919 * e)
        self.o.reset()
        self.g.reset()
        self.keys = KEYS[self.fam]
        self.coverage = coverage
        for e in range(E):
            for a in range(A):
                if coverage:
                    rs = {"teamSpirit": 0.0}
                    for k, key in enumerate(self.keys):
                        rs[key] = 16.0 ** k * 2.0 ** a
                    if self.fam == "tower":
                        rs["towerBuildingReward"] = 2.0 ** a / 256.0
                else:  # the scenario's own table, a non-zero team spirit and per-agent values
                    rs = {"teamSpirit": team_spirit[a]}
                    for k, key in enumerate(self.keys):
                        rs[key] = (k + 1) * (0.75 + 0.5 * a) * (-1.0 if k % 2 else 1.0)
                self.g.set_reward_shaping(e, a, rs)
                for key, v in rs.items():
                    self.O.orc_set_reward_shaping(self.o.h_, e, a, key.encode(), float(v))
        self.counts = {ev: 0 for ev in EVENTS[self.fam]}
        self.counts.update({"fall": 0} if self.fam in FALLS else {})
        if self.fam == "obstacles":
            self.counts["lava"] = 0
        if self.fam == "hexmemory":
            self.counts["all_good"] = 0
        self.early_ends = 0
        self.solved_pending = [False] * E
        self.dones = 0
        self.paid = 0  # non-zero rewards seen
        self.warps = 0
        self.checkpoints = 0
        self.states = [self.o.state(e) for e in range(E)]

    def close(self):
        self.o.close()
        self.g.close()

    # ---- views of the oracle's dumps
    def agent(self, e, a):
        st = self.states[e]
        return st[8 + AG * a: 8 + AG * (a + 1)]

    def objects(self, e):
        st = self.states[e]
        n = int(st[5])
        base = 8 + AG * self.A
        return st[base: base + 9 * n].reshape(n, 9)

    def level_rewards(self, e):
        """reward-object voxels of an Obstacles / Collect level (orc_get_level layout)"""
        L = self.o.level(e)
        i = 9 + 8 * int(L[0]) + 7 * int(L[1]) + 3 * int(L[2]) + 3 * self.A
        n = int(L[i + 1])
        return L[i + 2: i + 2 + 3 * n].reshape(n, 3)

    def alive(self, e):
        st = self.states[e]
        w = st[-6:].astype(np.int64)
        return [int(w[2 * k]) | (int(w[2 * k + 1]) << 24) for k in range(3)]

    # ---- warps: the oracle first, then the engine gets the oracle's floats
    def warp(self, e, a, x, y, z, yaw):
        self.O.orc_scen_warp(self.o.h_, e, a, float(x), float(y), float(z), float(yaw))
        st = self.o.state(e)
        ag = st[8 + AG * a: 8 + AG * (a + 1)]
        self.g.warp_agent(e, a, ag[0:3], ag[3:12])
        self.states[e] = st
        self.warps += 1

    def compare_state(self, e, tag):
        so, sg = self.o.state(e), self.g.state(e)
        assert so.shape == sg.shape, "%s env %d: state size %d vs %d" % (tag, e, so.size, sg.size)
        if not np.array_equal(so.view(np.uint32), sg.view(np.uint32)):
            bad = np.nonzero(so.view(np.uint32) != sg.view(np.uint32))[0]
            raise AssertionError("%s env %d: state words %s differ: oracle %s device %s" % (tag, e, bad[:8], so[bad[:8]], sg[bad[:8]]))
        assert np.array_equal(self.o.voxels(e), self.g.voxels(e)), "%s env %d: voxels" % (tag, e)

    def checkpoint(self, tag, frames=True):
        self.checkpoints += 1
        for e in range(self.E):
            self.compare_state(e, tag)
        if not frames:
            return
        self.O.orc_render_now(self.o.h_)
        a, b = self.o.obs(), np.array(self.g.obs())
        if self.fast:
            diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
            assert diff.max() <= 1, "%s: max RGB diff %d" % (tag, diff.max())
            assert float((diff == 0).mean()) > 0.999, tag
        else:
            assert np.array_equal(a, b), "%s: frames differ in %d bytes" % (tag, int((a != b).sum()))
        da, db = self.o.depth(), np.array(self.g.depth())
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32)), "%s: depth differs in %d pixels" % (tag, int((da != db).sum()))

    # ---- one tick on both sides
    def step(self, acts, tag, host=True):
        before = [s.copy() for s in self.states]
        self.o.step(acts)
        if host:
            self.g.step(acts)
            ro, rg = self.o.rewards(), np.array(self.g.rewards())
            assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "%s: rewards %s vs %s" % (tag, ro, rg)
            assert np.array_equal(self.o.dones(), np.array(self.g.dones())), "%s: dones" % tag
            assert np.array_equal(self.o.true_objectives().view(np.uint32), np.array(self.g.true_objectives()).view(np.uint32)), "%s: true objectives" % tag
        self.states = [self.o.state(e) for e in range(self.E)]
        self.count(before)
        return self.o.dones()

    def count(self, before):
        r = self.o.rewards().reshape(self.E, self.A)
        d = self.o.dones()
        self.paid += int((r != 0).sum())
        for e in range(self.E):
            if not d[e] and self.states[e][0] > before[e][0] + 2 * DT:
                self.solved_pending[e] = True  # doneWithTimer: the episode clock jumped to 0.3 s before its end
            if d[e]:
                self.dones += 1
                if self.solved_pending[e]:
                    self.early_ends += 1
                    if self.fam == "hexmemory":
                        self.counts["all_good"] += 1
                self.solved_pending[e] = False
            if self.fam == "tower" and not d[e] and self.states[e][4] != before[e][4]:
                self.counts["building"] += 1  # currBuildingZoneReward moved: an object was placed in the zone
            for a in range(self.A):
                b = before[e][8 + AG * a: 8 + AG * (a + 1)]
                n = self.states[e][8 + AG * a: 8 + AG * (a + 1)] if not d[e] else None
                fell = lava = False
                if n is not None and self.fam in FALLS:
                    fell = b[1] < -10 and n[1] > b[1] + 5
                    lava = self.fam == "obstacles" and not fell and b[1] >= -10 and math.hypot(n[0] - b[0], n[2] - b[2]) > 1.5 and not n[12:15].any()
                    self.counts["fall"] += int(fell)
                    if lava:
                        self.counts["lava"] += 1
                if not self.keys or not self.coverage:
                    continue
                v = float(r[e, a]) / 2.0 ** a
                if self.fam == "tower":
                    v = round(v)
                assert v == int(v) and v >= 0, "env %d agent %d: reward %r does not decode" % (e, a, float(r[e, a]))
                v = int(v)
                for k, ev in enumerate(EVENTS[self.fam]):
                    if self.fam == "tower" and ev == "building":
                        continue
                    c = (v >> (4 * k)) & 15
                    if self.fam == "collect" and ev == "bad" and fell:
                        c -= 1  # agentFell pays collectSingleBad
                    self.counts[ev] += c

    def table(self):
        return "%-16s A=%d E=%d warps=%d dones=%d early=%d paid=%d checkpoints=%d  %s" % (
            self.scenario, self.A, self.E, self.warps, self.dones, self.early_ends, self.paid, self.checkpoints,
            " ".join("%s=%d" % kv for kv in self.counts.items()))


# ------------------------------------------------------------------------------------------------ targeted warps
def beside_random_drawable(run, e, a, rng):
    """test_ref_shim.py's draw: next to a random object, reward, pillar or wall, random heading"""
    inst = run.o.instances(e)
    world = inst[inst[:, 2 + 12] < 400]
    special = world[world[:, 0] != 0]
    pool = special if len(special) and rng.random() < 0.6 else world
    m = pool[rng.integers(len(pool)), 2:]
    run.warp(e, a, m[12] + rng.uniform(-0.8, 0.8), m[13] + 1.2, m[14] + rng.uniform(-0.8, 0.8), rng.uniform(0, 2 * np.pi))


def facing_object(run, e, a, t, dist=1.0, rng=None):
    """stand `dist` from the centre of an object (at its height) facing it"""
    k = int(rng.integers(4))
    dx, dz = [(1, 0), (-1, 0), (0, 1), (0, -1)][k]
    run.warp(e, a, t[0] - dx * dist, t[1], t[2] - dz * dist, yaw_towards(dx, dz))


def cells(run, e, flag):
    v = run.o.voxels(e)
    return v[(v[:, 3] & flag) != 0, :3]


def plan_warps(run, e, rng, t):
    """warp the agents of env e towards the scenario's rare paths; returns {agent: action mask held for the next ticks}"""
    fam, A = run.fam, run.A
    hold = {}
    objs = run.objects(e)
    choice = rng.random()
    if fam in FALLS and choice < 0.08:  # below y = -20, or off the level's edge; an agent that carries something may put it down
        # out there, where it sinks to y = -30, outside the engine's dense grid beyond its margin
        a = int(rng.integers(A))
        p = run.agent(e, a)
        if rng.random() < 0.5:
            run.warp(e, a, p[0], -25.0, p[2], 0.0)
            hold[a] = 0
        else:
            v = run.o.voxels(e)
            run.warp(e, a, v[:, 0].min() - 6.0, p[1] + 1.0, p[2], 0.0)
            hold[a] = INTERACT if p[22] >= 0 else 0
        return hold
    if fam == "tower":
        for a in range(A):
            ag = run.agent(e, a)
            if ag[22] >= 0:  # carrying: into the building zone, then put it down
                L = run.o.level(e)
                x = rng.uniform(L[3] + 0.5, max(L[3] + 0.6, L[6] - 0.5))
                z = rng.uniform(L[5] + 0.5, max(L[5] + 0.6, L[8] - 0.5))
                run.warp(e, a, x, L[4] + 1.5, z, rng.uniform(0, 2 * np.pi))
                hold[a] = INTERACT if rng.random() < 0.7 else 0
            else:
                free = [o for o in objs if o[6] < 0]
                if free:
                    facing_object(run, e, a, free[int(rng.integers(len(free)))], rng=rng)
                    hold[a] = INTERACT
        return hold
    if fam == "obstacles":
        exits, lava = cells(run, e, 0x100), cells(run, e, 0x200)
        rewards = run.level_rewards(e)
        carrying = [a for a in range(A) if run.agent(e, a)[22] >= 0]
        if carrying and len(exits):
            a = carrying[0]
            c = exits[int(rng.integers(len(exits)))]
            run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, 0.0)
            hold[a] = 0
        elif choice < 0.3 and len(exits):  # all agents at once, on distinct cells of the exit's lowest layer
            low = exits[exits[:, 1] == exits[:, 1].min()]
            pick = rng.choice(len(low), size=A, replace=len(low) < A)
            for a in range(A):
                c = low[pick[a]]
                run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, 0.0)
                hold[a] = 0
        elif choice < 0.45 and len(exits):  # one agent only
            a = int(rng.integers(A))
            c = exits[int(rng.integers(len(exits)))]
            run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, 0.0)
            hold[a] = 0
        elif choice < 0.6 and len(lava):
            a = int(rng.integers(A))
            c = lava[int(rng.integers(len(lava)))]
            run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, 0.0)
            hold[a] = 0
        elif choice < 0.75 and len(rewards):
            a = int(rng.integers(A))
            c = rewards[int(rng.integers(len(rewards)))]
            run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, 0.0)
            hold[a] = 0
        elif len(objs) and (objs[:, 6] < 0).any():  # pick something up for the carried-to-exit bonus
            a = int(rng.integers(A))
            free = objs[objs[:, 6] < 0]
            facing_object(run, e, a, free[int(rng.integers(len(free)))], rng=rng)
            hold[a] = INTERACT
        else:
            beside_random_drawable(run, e, int(rng.integers(A)), rng)
        return hold
    if fam == "collect":
        rewards = run.level_rewards(e)
        alive = run.alive(e)
        live = [r for r in range(len(rewards)) if (alive[r >> 5] >> (r & 31)) & 1]
        rng.shuffle(live)
        for a in range(A):
            if live and rng.random() < 0.85:
                c = rewards[live.pop()]
                run.warp(e, a, c[0] + 0.5, c[1] + 0.5, c[2] + 0.5, rng.uniform(0, 2 * np.pi))
                hold[a] = 0
        return hold
    if fam == "sokoban":
        walls, goals = cells(run, e, 0x100), cells(run, e, 0x200)
        wallset = {tuple(c) for c in walls}
        goalset = {tuple(c) for c in goals}
        boxes = {tuple(np.floor(o[:3] / 2).astype(int)): o for o in objs}
        for a in range(A):
            if not boxes or rng.random() < 0.15:
                continue
            cell = list(boxes)[int(rng.integers(len(boxes)))]
            dirs = [(1, 0), (-1, 0), (0, 1), (0, -1)]
            to_goal = [d for d in dirs if (cell[0] + d[0], cell[1], cell[2] + d[1]) in goalset]
            if to_goal and cell not in goalset and rng.random() < 0.8:
                d = to_goal[0]
            else:
                d = dirs[int(rng.integers(4))]
            beyond = (cell[0] + d[0], cell[1], cell[2] + d[1])
            if beyond in wallset or beyond in boxes:
                continue
            c = boxes[cell]
            run.warp(e, a, c[0] - 1.5 * d[0], c[1] + 1.4, c[2] - 1.5 * d[1], yaw_towards(*d))
            hold[a] = INTERACT
        return hold
    if fam == "hexexplore":
        inst = run.o.instances(e)
        cones = inst[(inst[:, 0] == 3) & (inst[:, 2 + 12] < 400)]
        for a in range(A):
            if len(cones) and rng.random() < 0.5:
                m = cones[0, 2:]
                r = rng.uniform(0.0, 0.9)
                ang = rng.uniform(0, 2 * np.pi)
                run.warp(e, a, m[12] + r * math.cos(ang), run.agent(e, a)[1], m[14] + r * math.sin(ang), rng.uniform(0, 2 * np.pi))
                hold[a] = 0
            elif rng.random() < 0.5:
                beside_random_drawable(run, e, a, rng)
        return hold
    if fam == "hexmemory":
        inst = run.o.instances(e)
        items = inst[(inst[:, 0] >= 2) & (inst[:, 2 + 12] < 400)]
        for a in range(A):
            if len(items):
                m = items[int(rng.integers(len(items))), 2:]
                ang = rng.uniform(0, 2 * np.pi)
                run.warp(e, a, m[12] + 0.3 * math.cos(ang), m[13] + 0.6, m[14] + 0.3 * math.sin(ang), rng.uniform(0, 2 * np.pi))
                hold[a] = 0
        return hold
    if fam == "rearrange":  # agent 0 follows the scripted controller; the others are dropped next to things
        for a in range(1, A):
            beside_random_drawable(run, e, a, rng)
        if A == 1 and rng.random() < 0.2:
            beside_random_drawable(run, e, 0, rng)
        return hold
    for a in range(A):  # Empty
        beside_random_drawable(run, e, a, rng)
    return hold


def drive(run, ticks, rng, host=True, sync_every=0, check_every=25):
    """the warped, checked rollout; returns the number of ticks run"""
    E, A = run.E, run.A
    period = [5 + 2 * (e % 4) for e in range(E)]
    held = {}
    checkpoint_next = False
    for t in range(ticks):
        warped = False
        if host or (sync_every and t % sync_every == 0 and t > 0):
            for e in range(E):
                if (t + e) % period[e] == period[e] - 1:
                    for a, m in plan_warps(run, e, rng, t).items():
                        held[(e, a)] = (m, 2)
                    warped = True
            if warped and host:
                run.checkpoint("%s t=%d right after warps" % (run.scenario, t), frames=False)
        if run.fam == "rearrange":
            acts = np.concatenate([helpers.rearrange_controller(run.o, e, A) for e in range(E)]).astype(np.int32)
        else:
            acts = helpers.purposeful_actions(rng, E * A, t)
        for (e, a), (m, n) in list(held.items()):
            acts[e * A + a] = m
            held[(e, a)] = (m, n - 1)
            if n <= 1:
                del held[(e, a)]
        tag = "%s A=%d t=%d" % (run.scenario, A, t)
        d = run.step(acts, tag, host=host)
        if not host:
            run.g.step_device(run.dacts_ptr(acts))
            if sync_every and (t + 1) % sync_every == 0:
                run.g.sync()
                assert np.array_equal(run.o.rewards().view(np.uint32), np.array(run.g.rewards()).view(np.uint32)), tag
                assert np.array_equal(run.o.dones(), np.array(run.g.dones())), tag
                run.g.fetch_obs()
                run.checkpoint(tag + " sync")
            continue
        if checkpoint_next or d.any() or t % check_every == check_every - 1:
            run.checkpoint(tag)
        checkpoint_next = warped
    assert run.g.faults() == 0
    return ticks


def required_events(run):
    """the rules the run's levels offer"""
    fam = run.fam
    req = [ev for ev in EVENTS[fam] if ev != "abyss"]  # collectAbyss is declared but never paid (agentFell pays collectSingleBad)
    if fam == "obstacles":
        req = ["at_exit", "all_at_exit"]
        if run.seen_rewards:
            req.append("extra")
        if run.seen_objects:
            req.append("carried_to_exit")
        if run.seen_lava:
            req.append("lava")
    if fam in FALLS:
        req.append("fall")
    if fam == "hexmemory":
        req.append("all_good")
    return req


COVERAGE = [
    # scenario, A, E, ticks, seed
    ("TowerBuilding", 2, 12, 320, 101),
    ("ObstaclesEasy", 1, 10, 240, 102),
    ("ObstaclesMedium", 2, 10, 240, 103),
    ("ObstaclesHard", 3, 8, 240, 104),
    ("ObstaclesWalls", 2, 10, 240, 105),
    ("ObstaclesSteps", 1, 10, 240, 106),
    ("ObstaclesLava", 2, 10, 240, 107),
    ("Test", 2, 8, 160, 108),
    ("Collect", 2, 12, 320, 109),
    ("Collect", 8, 8, 240, 110),
    ("Sokoban", 2, 12, 240, 111),
    ("Rearrange", 1, 8, 450, 112),
    ("Rearrange", 2, 8, 450, 113),
    ("HexExplore", 2, 12, 200, 114),
    ("HexExplore", 1, 8, 200, 115),
    ("HexMemory", 1, 12, 260, 116),
    ("HexMemory", 2, 8, 260, 117),
    ("Empty", 2, 8, 120, 118),
]


def _coverage(scenario, A, E, ticks, seed):
    run = Run(scenario, E, A, seed, params={"episodeLengthSec": 30.0} if family(scenario) not in ("empty",) else {"episodeLengthSec": 6.0})
    try:
        run.seen_rewards = any(len(run.level_rewards(e)) for e in range(E)) if run.fam in ("obstacles", "collect") else False
        run.seen_objects = any(len(run.objects(e)) for e in range(E))
        run.seen_lava = any(len(cells(run, e, 0x200)) for e in range(E)) if run.fam == "obstacles" else False
        run.checkpoint("%s reset" % scenario)
        drive(run, ticks, np.random.default_rng(seed))
        print(run.table())
        missing = [ev for ev in required_events(run) if run.counts.get(ev, 0) == 0]
        assert not missing, "%s: rules that never fired: %s\n%s" % (scenario, missing, run.table())
        if run.fam in SOLVED:
            assert run.early_ends > 0, "%s: no solved rule ended an episode before its timer\n%s" % (scenario, run.table())
        return run.counts
    finally:
        run.close()


@pytest.mark.parametrize("scenario,A,E,ticks,seed", COVERAGE)
def test_every_rule_fires_and_matches_the_oracle(built, scenario, A, E, ticks, seed):
    _coverage(scenario, A, E, ticks, seed)


ONE_PUSH_ROOMS = """; 0
##########
#        #
#  $.    #
#        #
#   @    #
#        #
#    $   #
#    .   #
#        #
##########

; 1
##########
#        #
#   .$   #
#        #
#    @   #
#     $  #
#     .  #
#   $.   #
#        #
##########

; 2
##########
#        #
#  .     #
#  $     #
#      @ #
#   $.   #
#        #
#  .$    #
#        #
##########
"""


@pytest.mark.parametrize("A", [1, 2])
def test_sokoban_rooms_one_push_from_solved(built, tmp_path, monkeypatch, A):
    """Boxoban rooms in which every box is one push from a goal: boxes onto targets, off them again, and every room solved"""
    root = tmp_path / "boxoban" / "unfiltered" / "train"
    root.mkdir(parents=True)
    (root / "000.txt").write_text(ONE_PUSH_ROOMS)
    monkeypatch.setenv("BOXOBAN_LEVELS", str(tmp_path / "boxoban"))  # both sides read it when the env is constructed
    counts = _coverage("Sokoban", A, 10, 240, 120 + A)
    assert counts["all_on_target"] >= 3


def test_team_split_with_per_agent_values(built):
    """default reward tables, non-zero and per-agent team spirit: rewardTeam's split between the acting agent and the others"""
    for scenario, A in (("Collect", 3), ("ObstaclesHard", 2), ("TowerBuilding", 2), ("HexMemory", 2), ("Sokoban", 2)):
        run = Run(scenario, 8, A, 300 + A, params={"episodeLengthSec": 30.0}, coverage=False, team_spirit=[0.3, 0.7, 0.55][:A])
        try:
            run.seen_rewards = run.seen_objects = run.seen_lava = False
            drive(run, 160, np.random.default_rng(A), check_every=40)
            print("team split " + run.table())
            assert run.paid > 0, "%s: the team split was never exercised" % scenario
        finally:
            run.close()


def test_fast_shading_run_within_one_lsb(built):
    """the production fragment stage on a warped Collect run: frames within +-1 LSB, everything else bit-exact"""
    run = Run("Collect", 8, 2, 131, params={"episodeLengthSec": 30.0}, fast_shading=True)
    try:
        drive(run, 160, np.random.default_rng(5))
        print("fast shading " + run.table())
        assert run.counts["good"] > 0
    finally:
        run.close()


def test_async_path_with_warps_and_solved_ends(built):
    """mv_step_device with warps at the synchronisation points: rewards, dones, state, frames and depth at every sync, solved
    Collect episodes inside the run"""
    import torch

    run = Run("Collect", 8, 2, 141, params={"episodeLengthSec": 30.0})
    try:
        keep = []  # every action tensor stays alive until the run ends: the engine reads it in its own stream's order

        def dacts_ptr(acts):
            d = torch.from_numpy(np.ascontiguousarray(acts, np.int32)).cuda()
            torch.cuda.synchronize()
            keep.append(d)
            return d.data_ptr()

        run.dacts_ptr = dacts_ptr
        drive(run, 240, np.random.default_rng(9), host=False, sync_every=8)
        print("async " + run.table())
        assert run.early_ends > 0 and run.warps > 0
    finally:
        run.close()


def test_warp_hook_refusals(built):
    """mv_debug_warp_agent: call order (MV_ERR_STATE), bad indices / pointers / values (MV_ERR_ARG), and on any error nothing changes"""
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 2, 2, num_threads=2)
    L = capi.lib()
    pos, basis = np.float32([1, 2, 3]), np.eye(3, dtype=np.float32)
    with pytest.raises(capi.MegaverseError) as ei:
        g.warp_agent(0, 0, pos, basis)  # before reset
    assert ei.value.code == capi.MV_ERR_STATE
    g.seed(1)
    g.reset()
    for env, agent in ((-1, 0), (2, 0), (0, -1), (0, 2)):
        with pytest.raises(capi.MegaverseError) as ei:
            g.warp_agent(env, agent, pos, basis)
        assert ei.value.code == capi.MV_ERR_ARG
    for bad in (np.float32([np.nan, 2, 3]), np.float32([1, np.inf, 3])):
        with pytest.raises(capi.MegaverseError) as ei:
            g.warp_agent(0, 0, bad, basis)
        assert ei.value.code == capi.MV_ERR_ARG
    b2 = basis.copy(); b2[1, 1] = np.inf
    with pytest.raises(capi.MegaverseError):
        g.warp_agent(0, 0, pos, b2)
    assert L.mv_debug_warp_agent(g._h, 0, 0, None, basis.ctypes.data) == capi.MV_ERR_ARG
    g.step_begin(np.zeros(4, np.int32))
    with pytest.raises(capi.MegaverseError) as ei:
        g.warp_agent(0, 0, pos, basis)
    assert ei.value.code == capi.MV_ERR_STATE
    g.step_end()
    g2 = capi.Engine("Collect", 2, 2, num_threads=2)
    g2.seed(1); g2.reset(); g2.step(np.zeros(4, np.int32))
    for e in range(2):  # the refused calls changed nothing: the step matches an engine that never saw them
        assert np.array_equal(g.state(e).view(np.uint32), g2.state(e).view(np.uint32))
    g.warp_agent(1, 1, pos, basis)
    s = g.state(1)
    a = s[8 + AG: 8 + 2 * AG]
    assert np.array_equal(a[0:3], pos) and np.array_equal(a[3:12], basis.ravel()) and not a[12:16].any()
    assert np.array_equal(s[:8 + AG].view(np.uint32), g2.state(1)[:8 + AG].view(np.uint32))  # agent 0 untouched
    g.close(); g2.close()
