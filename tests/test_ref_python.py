"""The drop-in at the level a user touches it: the reference's own Python class megaverse.megaverse_env.MegaverseEnv (imported from
/root/reference, running on the reference's own pybind module and env library compiled in place on the Bullet stand-in -- tests/refpy.py)
wrote tests/golden/ref_python_env_golden.npz: seed(), reset(), step() with six-head actions, a reward-shaping change on the way.  The
same calls on this repository's MegaverseEnv (GPU suite) must return the same rewards, dones and true_reward infos; the CPU suite checks
the fixture against the reference class itself (where /root/reference is mounted) and against the oracle."""
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_python_env_golden.npz")
CASES = ["towerbuilding", "collect", "obstacleseasy", "hexmemory", "sokoban"]


def _replay(make_env, case):
    """make_env(scenario, E, A, params) -> object with the reference's MegaverseEnv interface"""
    g = np.load(GOLDEN)
    E, A, seed, T = (int(v) for v in g[case + "/meta"])
    N = E * A
    params = {str(k): float(v) for k, v in zip(g[case + "/param_keys"], g[case + "/param_vals"])} or None
    env = make_env(str(g[case + "/scenario"]), E, A, params)
    assert env.num_agents == N and env.num_envs == E and env.num_agents_per_env == A and env.is_multiagent
    assert [s.n for s in env.action_space.spaces] == [3, 3, 3, 2, 2, 3]
    assert tuple(env.observation_space.shape) == (3, 72, 128)
    keys = [str(k) for k in g[case + "/shaping_keys"]]
    default = env.get_default_reward_shaping()
    assert sorted(default) == keys
    assert np.array_equal(np.array([default[k] for k in keys], np.float32), g[case + "/shaping_default"])
    env.seed(seed)
    obs = env.reset()
    assert len(obs) == N and obs[0].shape == (3, 72, 128) and obs[0].dtype == np.uint8
    change_t, change_actor = (int(v) for v in g[case + "/change"])
    acts, rew, done, true_reward = g[case + "/actions"], g[case + "/rewards"], g[case + "/dones"], g[case + "/true_reward"]
    for t in range(T):
        if t == change_t:
            rs = dict(env.get_current_reward_shaping(change_actor))
            rs[str(g[case + "/change_key"])] = float(g[case + "/change_val"])
            env.set_reward_shaping(rs, change_actor)
        obs, r, d, infos = env.step([[int(x) for x in a] for a in acts[t]])
        assert len(obs) == N and len(r) == N and len(d) == N and len(infos) == N
        assert np.array_equal(np.asarray(r, np.float32).view(np.uint32), rew[t].view(np.uint32)), "%s: rewards at tick %d: %s, reference %s" % (case, t, r, rew[t])
        assert [bool(x) for x in d] == [bool(x) for x in done[t]], "%s: dones at tick %d" % (case, t)
        for i, inf in enumerate(infos):
            if done[t, i]:
                assert np.float32(inf["true_reward"]) == true_reward[t, i], "%s: true_reward at tick %d actor %d" % (case, t, i)
            else:
                assert inf == {}, "%s: info of a running env at tick %d" % (case, t)
    final = np.array([[env.get_current_reward_shaping(i)[k] for k in keys] for i in range(N)], np.float32)
    assert np.array_equal(final, g[case + "/shaping_final"]), "%s: reward shaping after the run" % case
    env.close()


@pytest.mark.parametrize("case", CASES)
def test_reference_python_class_reproduces_its_golden(built, case):
    """the fixture is what the reference's class returns today (guards the fixture and the replay code); needs /root/reference"""
    import refpy

    if not refpy.available():
        pytest.skip("/root/reference absent")
    RefEnv = refpy.reference_env_class()
    _replay(lambda s, E, A, p: RefEnv(s, num_envs=E, num_agents_per_env=A, num_simulation_threads=1, use_vulkan=True, params=p), case)


class _OracleEnv:
    """the oracle behind the same interface (six-head actions through helpers.encode), for the CPU suite on boxes without /root/reference"""

    def __init__(self, scenario, E, A, params):
        import orc
        from types import SimpleNamespace

        self.o = orc.Oracle(scenario, E, A, params=params, render=False)
        self.num_envs, self.num_agents_per_env, self.num_agents, self.is_multiagent = E, A, E * A, True
        self.action_space = SimpleNamespace(spaces=[SimpleNamespace(n=n) for n in (3, 3, 3, 2, 2, 3)])
        self.observation_space = SimpleNamespace(shape=(3, 72, 128))
        self._default = self.get_current_reward_shaping(0)

    def get_default_reward_shaping(self):
        return self._default

    def get_current_reward_shaping(self, actor):
        import ctypes as C

        import orc

        out = {}
        for k in ("teamSpirit", "towerPickedUpObject", "towerVisitedBuildingZoneWithObject", "towerBuildingReward", "collectSingleGood", "collectSingleBad", "collectAll",
                  "collectAbyss", "obstaclesAgentAtExit", "obstaclesAllAgentsAtExit", "obstaclesExtraReward", "obstaclesAgentCarriedObjectToExit", "sokobanBoxOnTarget",
                  "sokobanBoxLeavesTarget", "sokobanAllBoxesOnTarget", "memoryCollectGood", "memoryCollectBad", "exploreSolved",
                  "rearrangeOneMoreObjectCorrectPosition", "rearrangeAllObjectsCorrectPosition"):
            v = C.c_float()
            if orc.lib().orc_get_reward_shaping(self.o.h_, actor // self.num_agents_per_env, actor % self.num_agents_per_env, k.encode(), C.byref(v)) == 0:
                out[k] = v.value
        return out

    def set_reward_shaping(self, rs, actor):
        import orc

        for k, v in rs.items():
            orc.lib().orc_set_reward_shaping(self.o.h_, actor // self.num_agents_per_env, actor % self.num_agents_per_env, k.encode(), float(v))

    def seed(self, s):
        self.o.seed(s)

    def _obs(self):
        return [np.zeros((3, 72, 128), np.uint8)] * self.num_agents

    def reset(self):
        self.o.reset()
        return self._obs()

    def step(self, actions):
        import helpers

        self.o.step(np.array([helpers.encode(a) for a in actions], np.int32))
        d = np.repeat(self.o.dones(), self.num_agents_per_env)
        to = self.o.true_objectives()
        infos = [dict(true_reward=float(to[i])) if d[i] else {} for i in range(self.num_agents)]
        return self._obs(), list(self.o.rewards()), [bool(x) for x in d], infos

    def close(self):
        self.o.close()


@pytest.mark.parametrize("case", CASES)
def test_product_default_reward_shaping_matches_the_reference_golden(built, case):
    """the tables the engine is built from (host-only accessor, no GPU) hold the default reward shaping the reference's class returned,
    key for key and bit for bit"""
    import ctypes as C

    from megaverse_b200 import capi

    g = np.load(GOLDEN)
    L = capi.lib()
    L.mv_debug_defaults.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
    buf = C.create_string_buffer(8192)
    assert L.mv_debug_defaults(str(g[case + "/scenario"]).encode(), buf, 8192) > 0
    ours = dict(ln[2:].split("=") for ln in buf.value.decode().splitlines() if ln.startswith("R "))
    ref = {str(k): "%08x" % v for k, v in zip(g[case + "/shaping_keys"], g[case + "/shaping_default"].view(np.uint32))}
    assert ours == ref, "reward shaping:\nreference %s\nproduct   %s" % (ref, ours)


@pytest.mark.parametrize("case", CASES)
def test_oracle_replays_the_reference_python_golden(built, case):
    _replay(_OracleEnv, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_our_python_env_replays_the_reference_python_golden(built, case):
    """this repository's MegaverseEnv (megaverse_b200/megaverse_env.py over the pybind module over the C ABI over the CUDA engine)"""
    from megaverse_b200 import MegaverseEnv

    _replay(lambda s, E, A, p: MegaverseEnv(s, num_envs=E, num_agents_per_env=A, num_simulation_threads=2, use_vulkan=True, params=p), case)
