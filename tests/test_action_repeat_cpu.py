"""Action repeat (option "action_repeat") without a GPU: the option refuses a null handle, the header documents it with its range, and
MegaverseEnv takes it as a keyword-only argument beside final_observation.  The range and the set-after-reset refusal need an engine and
are checked in test_action_repeat_gpu.py."""
import inspect
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_action_repeat_refuses_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    for k in (0, 1, 2, 4, 5):
        assert L.mv_set_option(None, b"action_repeat", k) == capi.MV_ERR_ARG


def test_action_repeat_is_documented(built):
    with open(os.path.join(ROOT, "include", "megaverse_b200.h")) as f:
        header = f.read()
    assert '"action_repeat" (1..4, before the first reset' in header
    assert "3k ticks" in header


def test_megaverse_env_keyword(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    params = inspect.signature(MegaverseEnv.__init__).parameters
    positional = [n for n, p in params.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == ["self", "scenario_name", "num_envs", "num_agents_per_env", "num_simulation_threads", "use_vulkan", "params"]
    assert params["action_repeat"].kind == inspect.Parameter.KEYWORD_ONLY and params["action_repeat"].default == 1
    assert params["final_observation"].kind == inspect.Parameter.KEYWORD_ONLY
