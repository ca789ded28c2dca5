"""Reference side of the reward-component tests (option "reward_components").

The key-to-slot table is restated here from the reference's scenario headers (the MV_R_* numbering of csrc/mv_types.h); the tests pin
it against mv_reward_component_keys.

The per-slot columns come from the oracle itself, unchanged.  A reward is sum of terms weight[slot] * ..., and weights steer no game
rule: an oracle twin whose shaping keeps teamSpirit and slot k's weight and sets every other weight to 0 pays exactly slot k's terms, in
the same order, plus exact zeros (0 * x = +-0, and x + +-0 = x).  So its reward is slot k's column bit for bit: the terms summed from
0.0f in event order within a tick.  One twin per slot, stepped with the same actions, gives every column."""
import numpy as np

import orc

R_COUNT = 8

# scenario family -> {shaping key: slot}
KEY_SLOTS = {
    "tower": {"towerPickedUpObject": 1, "towerVisitedBuildingZoneWithObject": 2, "towerBuildingReward": 3},
    "collect": {"collectSingleGood": 1, "collectSingleBad": 2, "collectAll": 3, "collectAbyss": 4},
    "obstacles": {"obstaclesAgentAtExit": 1, "obstaclesAllAgentsAtExit": 2, "obstaclesExtraReward": 3, "obstaclesAgentCarriedObjectToExit": 4},
    "rearrange": {"rearrangeOneMoreObjectCorrectPosition": 1, "rearrangeAllObjectsCorrectPosition": 2},
    "sokoban": {"sokobanBoxOnTarget": 1, "sokobanBoxLeavesTarget": 2, "sokobanAllBoxesOnTarget": 3},
    "hexexplore": {"exploreSolved": 1},
    "hexmemory": {"memoryCollectGood": 1, "memoryCollectBad": 2},
    "empty": {},
}
# every registered name
NAMES = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
         "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava", "Test"]


def family(scenario):
    n = scenario.lower()
    if n.startswith("obstacles") or n == "test":
        return "obstacles"
    return {"towerbuilding": "tower"}.get(n, n)


def keys8(scenario):
    """the restated table as mv_reward_component_keys lays it out: slot k's key, None for slot 0 and unused slots"""
    out = [None] * R_COUNT
    for k, s in KEY_SLOTS[family(scenario)].items():
        out[s] = k
    return out


def random_shaping(rng, scenario, A, team_spirit=0.3):
    """per-agent shaping dicts: every key of the scenario at a random signed weight, team spirit as given"""
    out = []
    for _ in range(A):
        d = {"teamSpirit": float(team_spirit)}
        for k in KEY_SLOTS[family(scenario)]:
            d[k] = float(np.float32(rng.choice([-1.0, 1.0]) * rng.uniform(0.05, 3.0)))
        out.append(d)
    return out


class SlotOracles:
    """an oracle of `scenario` (E envs, A agents) and one masked twin per slot the scenario has a key for; every method acts on all of them.
    shaping: per view (env * A + agent) a dict, or None for the scenario's defaults"""

    def __init__(self, scenario, E, A, params=None, shaping=None):
        self.scenario, self.E, self.A, self.N = scenario, E, A, E * A
        self.main = orc.Oracle(scenario, E, A, params=params, render=False)
        self.slots = sorted(KEY_SLOTS[family(scenario)].values())
        self.twins = {s: orc.Oracle(scenario, E, A, params=params, render=False) for s in self.slots}
        key_of = {s: k for k, s in KEY_SLOTS[family(scenario)].items()}
        L = orc.lib()
        for v in range(self.N):
            e, a = divmod(v, A)
            full = dict(shaping[v]) if shaping is not None else self.defaults(e, a)
            for key, val in full.items():
                L.orc_set_reward_shaping(self.main.h_, e, a, key.encode(), float(val))
            for s, o in self.twins.items():
                for key, val in full.items():
                    keep = key == "teamSpirit" or key == key_of[s]
                    L.orc_set_reward_shaping(o.h_, e, a, key.encode(), float(val) if keep else 0.0)

    def defaults(self, e, a):
        import ctypes as C

        out = {}
        for key in ["teamSpirit"] + list(KEY_SLOTS[family(self.scenario)]):
            v = C.c_float()
            orc.lib().orc_get_reward_shaping(self.main.h_, e, a, key.encode(), C.byref(v))
            out[key] = v.value
        return out

    def all(self):
        return [self.main] + list(self.twins.values())

    def close(self):
        for o in self.all():
            o.close()

    def seed_env(self, e, s):
        for o in self.all():
            o.seed_env(e, s)

    def reset(self):
        for o in self.all():
            o.reset()

    def step(self, acts):
        for o in self.all():
            o.step(acts)
        d = self.main.dones()
        for o in self.twins.values():
            assert np.array_equal(o.dones(), d), "a masked twin left the main oracle's episode"

    def rewards(self):
        return self.main.rewards()

    def dones(self):
        return self.main.dones()

    def columns(self):
        """float32 [N, 8]: this tick's reward of every view split by slot"""
        c = np.zeros((self.N, R_COUNT), dtype=np.float32)
        for s, o in self.twins.items():
            c[:, s] = o.rewards()
        return c


class Totals:
    """the caller's side of the episode rows: the step rows summed in call order from 0.0f per view, the sum handed over at an end"""

    def __init__(self, N, A):
        self.A = A
        self.run = np.zeros((N, R_COUNT), dtype=np.float32)
        self.episode = np.zeros((N, R_COUNT), dtype=np.float32)

    def add(self, step, dones, tag=""):
        """one delivered call: step rows [N, 8], dones [E]; returns the views whose episode rows changed"""
        self.run = (self.run + np.asarray(step, dtype=np.float32)).astype(np.float32)
        ended = np.repeat(np.asarray(dones) != 0, self.A)
        self.episode[ended] = self.run[ended]
        self.run[ended] = 0.0
        return ended

    def restart(self, envs):
        for e in envs:
            self.run[e * self.A:(e + 1) * self.A] = 0.0

    def check(self, episode, tag):
        got = np.asarray(episode, dtype=np.float32)
        assert np.array_equal(got.view(np.uint32), self.episode.view(np.uint32)), "%s: episode rows %s vs %s" % (
            tag, got[np.any(got != self.episode, axis=1)][:4], self.episode[np.any(got != self.episode, axis=1)][:4])


def same_bits(a, b, tag):
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    if not np.array_equal(a.view(np.uint32), b.view(np.uint32)):
        bad = np.argwhere(a.view(np.uint32) != b.view(np.uint32))[:6]
        raise AssertionError("%s: %d values differ, first at %s: %s vs %s" % (tag, len(np.argwhere(a != b)), bad.tolist(),
                                                                          [float(a[tuple(i)]) for i in bad], [float(b[tuple(i)]) for i in bad]))
