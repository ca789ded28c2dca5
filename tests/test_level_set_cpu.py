"""Level sets without a GPU: the pick hash (mv_level_set_pick) and the definition of "level j of a set seeded s" that the GPU tests rely
on -- the first level of a generator seeded s + j, which the oracle reaches with seed_env(0, s + j); reset()."""
import numpy as np
import pytest

import orc


def _pick(seed, episode, count):
    from megaverse_b200 import capi

    return capi.level_set_pick(seed, episode, count)


def test_pick_is_deterministic_and_in_range(built):
    rng = np.random.default_rng(0)
    for count in (1, 2, 7, 1000, 65536):
        for seed, ep in zip(rng.integers(0, 2**32, 500), rng.integers(0, 100000, 500)):
            j = _pick(int(seed), int(ep), count)
            assert 0 <= j < count
            assert j == _pick(int(seed), int(ep), count)
    assert _pick(5, 3, 0) == 0 and _pick(5, 3, -4) == 0  # nothing to choose from: never an index beyond the bank


def test_pick_covers_a_set_uniformly(built):
    """10^5 (seed, episode) pairs over a 64-level set: every level is hit, chi-square against uniform is unremarkable (63 degrees of
    freedom: mean 63, the 99.99th percentile is 117)"""
    L = 64
    counts = np.zeros(L, dtype=np.int64)
    for seed in range(1000):
        for ep in range(100):
            counts[_pick(1000 + seed, ep, L)] += 1
    assert counts.min() > 0
    expect = counts.sum() / L
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    assert chi2 < 117.0, chi2


@pytest.mark.parametrize("L", [7, 64, 1000])
def test_pick_has_no_fixed_stride(built, L):
    """consecutive episodes of one seed, and one episode of consecutive seeds (how mv_seed_env is usually called: 42 + env): the step from
    one pick to the next takes many values, none dominates, and neighbours are uncorrelated"""
    n = 4000
    for seq in ([_pick(42, ep, L) for ep in range(n)], [_pick(42 + e, 0, L) for e in range(n)], [_pick(42 + e, 5, L) for e in range(n)]):
        seq = np.array(seq)
        stride = np.bincount((seq[1:] - seq[:-1]) % L, minlength=L)
        assert (stride > 0).sum() >= min(L, 400) * 0.9
        assert stride.max() < 4.0 * n / L + 20
        r = np.corrcoef(seq[:-1], seq[1:])[0, 1]
        assert abs(r) < 0.06, r


@pytest.mark.parametrize("scenario,A", [("Collect", 2), ("TowerBuilding", 1), ("ObstaclesHard", 2)])
def test_level_j_is_the_oracles_first_level_of_seed_s_plus_j(built, scenario, A):
    from megaverse_b200 import capi

    s = 100
    o = orc.Oracle(scenario, 1, A, render=False)
    for j in (0, 1, 5):
        o.seed_env(0, s + j)
        o.reset()
        want = o.level(0)
        got = capi.generate_level(scenario, A, s + j, 0)
        assert np.array_equal(got[:want.size], want), "%s: level %d" % (scenario, j)
    o.close()


def test_exports(built):
    from megaverse_b200 import capi

    for name in ("mv_level_ids", "mv_level_ids_device", "mv_next_levels_device", "mv_set_next_levels", "mv_level_set_pick"):
        assert name in capi.EXPORTS and hasattr(capi.lib(), name)
