"""Replaceable level-set rows without a GPU: the exports and their ctypes signatures, null handles, the argument checks of
MegaverseEnv.replace_levels / level_seeds, and `pick_with_probe`, the restatement of the step kernel's pick that the GPU tests predict
picks with: the hash's row, or the first pickable row after it (mod L) when that row is being replaced."""
import ctypes as C

import pytest

from test_level_set_cpu import _pick


def pick_with_probe(seed, episode, L, pickable, next_level=-1):
    """(level, entry left) of the flip at the start of episode `episode` of an env with pick seed `seed` in a block of L rows whose
    pickable flags are pickable[0..L): a next-level entry in [0, L) naming a pickable row is used and cleared (-1); any other entry is
    left as it is, and the hash's row is probed forward to the first pickable one"""
    from megaverse_b200 import capi

    if 0 <= next_level < L and pickable[next_level]:
        return next_level, -1
    j = capi.level_set_pick(seed, episode, L)
    for _ in range(L):
        if pickable[j]:
            return j, next_level
        j = (j + 1) % L
    raise AssertionError("a block with no pickable row")


def test_exports_and_signatures(built):
    from megaverse_b200 import capi

    L = capi.lib()
    for name in ("mv_replace_levels", "mv_level_rows"):
        assert name in capi.EXPORTS and hasattr(L, name)
    assert L.mv_replace_levels.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    assert L.mv_level_rows.argtypes == [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]


def test_null_handles(built):
    from megaverse_b200 import capi

    L = capi.lib()
    rows = (C.c_int32 * 1)(0)
    s, r = C.c_void_p(), C.c_void_p()
    assert L.mv_replace_levels(None, rows, rows, 1) == capi.MV_ERR_ARG
    assert L.mv_replace_levels(None, None, None, 0) == capi.MV_ERR_ARG
    assert L.mv_level_rows(None, C.byref(s), C.byref(r)) == capi.MV_ERR_ARG
    assert L.mv_level_rows(None, None, None) == capi.MV_ERR_ARG


def test_pick_with_probe_restatement(built):
    L = 8
    everything = [True] * L
    for seed in range(50):
        for ep in range(5):
            assert pick_with_probe(seed, ep, L, everything) == (_pick(seed, ep, L), -1)
    j = _pick(3, 1, L)
    flags = [True] * L
    flags[j] = False
    assert pick_with_probe(3, 1, L, flags) == ((j + 1) % L, -1)
    flags[(j + 1) % L] = False
    assert pick_with_probe(3, 1, L, flags) == ((j + 2) % L, -1)
    only = [False] * L
    only[(j + L - 1) % L] = True  # the probe wraps around the block
    assert pick_with_probe(3, 1, L, only) == ((j + L - 1) % L, -1)
    # an entry naming a retiring row stays and the hash probes; one naming a pickable row is used once; one outside the set is ignored
    assert pick_with_probe(3, 1, L, flags, next_level=j) == ((j + 2) % L, j)
    assert pick_with_probe(3, 1, L, flags, next_level=(j + 3) % L) == ((j + 3) % L, -1)
    assert pick_with_probe(3, 1, L, everything, next_level=L + 4) == (_pick(3, 1, L), L + 4)


class _FakeGym:
    """records what MegaverseEnv passes down"""

    def __init__(self, B):
        self.calls = []
        self.B = B

    def replace_levels(self, rows, seeds):
        self.calls.append((list(rows), list(seeds)))

    def get_level_rows(self):
        import numpy as np

        return np.arange(100, 100 + self.B, dtype=np.int32), np.zeros(self.B, dtype=np.uint8)


def _env(scenarios, num_levels):
    from megaverse_b200.megaverse_env import MegaverseEnv

    env = MegaverseEnv.__new__(MegaverseEnv)  # the argument checks need no engine
    env.scenarios = [s.casefold() for s in scenarios]
    env.num_levels = num_levels
    env.env = _FakeGym(len(dict.fromkeys(env.scenarios)) * (num_levels or 0))
    return env


def test_python_argument_checks(built):
    single = _env(["collect"] * 3, 4)
    single.replace_levels([1, 3], [77, 78])
    assert single.env.calls[-1] == ([1, 3], [77, 78])
    assert single.level_seeds() == [100, 101, 102, 103]
    with pytest.raises(ValueError):
        single.replace_levels([4], [1])  # outside the set
    with pytest.raises(ValueError):
        single.replace_levels([-1], [1])
    with pytest.raises(ValueError):
        single.replace_levels([0, 1], [1])  # lengths differ
    with pytest.raises(ValueError):
        single.replace_levels([0], [1], scenario="sokoban")  # not in the batch
    assert len(single.env.calls) == 1
    mixed = _env(["Collect", "TowerBuilding", "collect"], 4)
    with pytest.raises(ValueError):
        mixed.replace_levels([0], [1])  # which block?
    with pytest.raises(ValueError):
        mixed.level_seeds()
    mixed.replace_levels([0, 2], [5, 6], scenario="TowerBuilding")
    assert mixed.env.calls[-1] == ([4, 6], [5, 6])
    assert mixed.level_seeds("towerbuilding") == [104, 105, 106, 107]
    assert mixed.level_seeds("Collect") == [100, 101, 102, 103]
    for fn in (lambda e: e.replace_levels([0], [1]), lambda e: e.level_seeds()):
        with pytest.raises(ValueError):
            fn(_env(["collect"], None))  # no level set
