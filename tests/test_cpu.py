"""CPU-only tests (`-m "not gpu"`): the oracle against the reference's own pins, host level generation against the oracle,
the libstdc++ hash-set order emulation, and the C ABI's exported symbols.  No compute call needs a GPU here."""
import ctypes as C
import os
import sys
import subprocess

import numpy as np
import pytest

import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol(built):
    """every function include/megaverse_b200.h declares is exported by the in-tree .so, and the list in capi.py is complete"""
    import re
    from megaverse_b200 import capi

    hdr = open(os.path.join(ROOT, "include", "megaverse_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(mv_[a-z0-9_]+)\s*\(", hdr)))
    assert sorted(capi.EXPORTS) == declared
    L = C.CDLL(capi.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), name


def test_library_holds_sm90a_code(built):
    """the kernels are compiled for the H100 (sm_90a) and for nothing else: a cubin for another architecture does not load there"""
    import shutil
    from megaverse_b200 import capi

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "--list-elf", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    archs = sorted(set(ln.rsplit(".", 2)[-2] for ln in out.splitlines() if ln.strip().endswith(".cubin")))
    assert archs == ["sm_90a"], out


def test_no_cpu_fallback(built):
    """without a CUDA device the product must fail loudly (no oracle / CPU path behind the ABI)"""
    import torch
    from megaverse_b200 import capi

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(capi.MegaverseError) as ei:
        capi.Engine("TowerBuilding", 1, 1)
    assert ei.value.code == capi.MV_ERR_CUDA
    with pytest.raises(capi.MegaverseError) as ei:
        capi.Engine("NoSuchScenario", 1, 1)
    assert ei.value.code == capi.MV_ERR_ARG


def test_argument_errors_are_reported_not_fatal(built):
    """argument validation happens before any CUDA call, so it is testable without a device: status code + mv_last_error instead of the
    reference's TLOG(FATAL) -> exit(-1)"""
    from megaverse_b200 import capi

    for args, kwargs, needle in (
        (("NoSuchScenario", 1, 1), {}, "unknown scenario"),
        (("TowerBuilding", 0, 1), {}, "num_envs"),
        (("TowerBuilding", 1, 99), {}, "num_envs"),
        (("TowerBuilding", 1, 1, 100, 72), {}, "render size"),
        (("TowerBuilding", 1, 1), {"params": {"useUIRewardIndicators": 1.0}}, "useUIRewardIndicators"),
    ):
        with pytest.raises(capi.MegaverseError) as ei:
            capi.Engine(*args, **kwargs)
        assert ei.value.code == capi.MV_ERR_ARG, (args, ei.value)
        assert needle in str(ei.value), (args, ei.value)


def test_product_does_not_link_or_import_the_oracle(built):
    from megaverse_b200 import capi

    out = subprocess.run(["ldd", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "liborc" not in out
    for dirpath, _, files in os.walk(os.path.join(ROOT, "megaverse_b200")):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".h", ".hpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle/" not in txt.replace("oracle/ref_shim/dump_primitives.cpp", "").replace("oracle/orc_api.cpp", "").replace("`make -C oracle meshes`", ""), f
                assert "liborc" not in txt and "import orc" not in txt, f


def test_action_encoding(built):
    """megaverse.cpp:100-116 / env.hpp:22-42: Left=1<<1 ... LookUp=1<<10"""
    from megaverse_b200 import capi

    assert capi.encode_action([1, 0, 0, 0, 0, 0]) == 1 << 1
    assert capi.encode_action([2, 0, 0, 0, 0, 0]) == 1 << 2
    assert capi.encode_action([0, 1, 0, 0, 0, 0]) == 1 << 3
    assert capi.encode_action([0, 2, 0, 0, 0, 0]) == 1 << 4
    assert capi.encode_action([0, 0, 1, 0, 0, 0]) == 1 << 5
    assert capi.encode_action([0, 0, 2, 0, 0, 0]) == 1 << 6
    assert capi.encode_action([0, 0, 0, 1, 0, 0]) == 1 << 7
    assert capi.encode_action([0, 0, 0, 0, 1, 0]) == 1 << 8
    assert capi.encode_action([0, 0, 0, 0, 0, 1]) == 1 << 9
    assert capi.encode_action([0, 0, 0, 0, 0, 2]) == 1 << 10
    rng = np.random.default_rng(0)
    for _ in range(200):
        heads = [int(rng.integers(0, s)) for s in helpers.SIZES]
        assert capi.encode_action(heads) == helpers.encode(heads)


def test_unordered_set_order_emulation(built):
    """csrc/bzset.h reproduces the iteration order of a real std::unordered_set<VoxelCoords> (insert / erase / clear,
    rehashes 1->13->29->59->127): the order TowerBuilding's float reward sum runs in"""
    import orc
    from megaverse_b200 import capi

    L = orc.lib()
    L.orc_unordered_set_order.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    rng = np.random.default_rng(0)
    for _ in range(200):
        ops, present = [], []
        for _ in range(int(rng.integers(1, 220))):
            r = rng.random()
            if r < 0.6 or not present:
                v = (int(rng.integers(0, 30)), int(rng.integers(0, 8)), int(rng.integers(0, 25)))
                ops.append((0,) + v)
                if v not in present:
                    present.append(v)
            elif r < 0.95:
                v = present[int(rng.integers(0, len(present)))]
                ops.append((1,) + v)
                present.remove(v)
            else:
                ops.append((2, 0, 0, 0))
                present = []
            if len(present) > 110:
                ops.append((2, 0, 0, 0))
                present = []
        ops = np.array(ops, dtype=np.int32)
        out = np.zeros(3 * 256, dtype=np.int32)
        k = L.orc_unordered_set_order(ops.ctypes.data, len(ops), out.ctypes.data, out.size)
        assert np.array_equal(out[: k * 3].reshape(k, 3), capi.bzset_order(ops))


@pytest.mark.parametrize("scenario,num_agents", [("TowerBuilding", 1), ("TowerBuilding", 4), ("ObstaclesHard", 1), ("ObstaclesEasy", 2), ("ObstaclesMedium", 3),
                                                 ("ObstaclesWalls", 1), ("ObstaclesSteps", 2), ("ObstaclesLava", 1), ("Collect", 1), ("Collect", 4), ("Rearrange", 1), ("Rearrange", 3), ("Sokoban", 1), ("Sokoban", 4), ("HexExplore", 1), ("HexExplore", 3), ("HexMemory", 1), ("HexMemory", 4)])
def test_level_generation_matches_oracle(built, scenario, num_agents):
    """the product's flat host level generator against the oracle's reference-style one: same RNG draws, same merged
    boxes in the same order, same objects, spawn cells and spawn yaw bits -- over consecutive episodes of one stream"""
    import orc
    from megaverse_b200 import capi

    for seed in range(40, 70):
        o = orc.Oracle(scenario, 1, num_agents, render=False)
        o.seed_env(0, seed)
        for episode in range(3):
            o.reset()
            want = o.level(0)
            got = capi.generate_level(scenario, num_agents, seed, episode)
            n = len(want)
            assert np.array_equal(want, got[:n]), "%s seed %d episode %d: first diff at %s" % (scenario, seed, episode, np.nonzero(want != got[:n])[0][:5])
            st = o.state(0)
            basis = np.concatenate([st[8 + 26 * a + 3: 8 + 26 * a + 12] for a in range(num_agents)]).view(np.int32)
            assert np.array_equal(basis, got[n:]), "spawn basis seed %d episode %d" % (seed, episode)
        o.close()


def test_oracle_reference_pins(built):
    """the pins the reference's own tests hold for this path (SURVEY.md 8c)"""
    import orc

    L = orc.lib()
    # src/test/src/voxel_grid_tests.cpp:25  getCoords({1.5,2.3,3.2}) == {1,2,3}  -- exercised through the pick-up voxel maths:
    # the oracle's toVoxel is lround(floor(v)); check the documented example and a negative coordinate
    L.orc_to_voxel.argtypes = [C.c_float, C.c_float, C.c_float, C.c_void_p]
    out = np.zeros(3, dtype=np.int32)
    L.orc_to_voxel(1.5, 2.3, 3.2, out.ctypes.data)
    assert out.tolist() == [1, 2, 3]
    L.orc_to_voxel(-0.5, -1.0, 0.999, out.ctypes.data)
    assert out.tolist() == [-1, -1, 0]
    # megaverse/tests/test_env.py:42-53  same seed => identical first observation
    a = orc.Oracle("TowerBuilding", 2, 2); b = orc.Oracle("TowerBuilding", 2, 2)
    a.seed(42); b.seed(42); a.reset(); b.reset()
    assert np.array_equal(a.obs(), b.obs())
    c = orc.Oracle("TowerBuilding", 2, 2); c.seed(43); c.reset()
    assert not np.array_equal(a.obs(), c.obs())
    # megaverse/tests/test_env.py:123-140  reward shaping is per actor
    v = C.c_float()
    assert L.orc_get_reward_shaping(a.h_, 0, 0, b"teamSpirit", C.byref(v)) == 0 and abs(v.value - 0.1) < 1e-7
    L.orc_set_reward_shaping(a.h_, 0, 1, b"teamSpirit", 0.5)
    L.orc_get_reward_shaping(a.h_, 0, 0, b"teamSpirit", C.byref(v)); assert abs(v.value - 0.1) < 1e-7
    L.orc_get_reward_shaping(a.h_, 0, 1, b"teamSpirit", C.byref(v)); assert abs(v.value - 0.5) < 1e-7
    # libstdc++ stream pins probed by SURVEY.md Appendix C
    L.orc_rng_probe.argtypes = [C.c_void_p]
    pr = np.zeros(3, dtype=np.float64)
    L.orc_rng_probe(pr.ctypes.data)
    assert pr[0] == 1608637542 and pr[1] == 3 and abs(pr[2] - 0.796543002) < 1e-8
    for x in (a, b, c):
        x.close()


def test_oracle_golden_trajectory(built):
    """the oracle against committed golden vectors (tests/golden/tower_golden.npz, made by tests/golden/make_golden.py)"""
    import orc

    path = os.path.join(ROOT, "tests", "golden", "tower_golden.npz")
    g = np.load(path)
    o = orc.Oracle("TowerBuilding", int(g["E"]), int(g["A"]))
    o.seed(int(g["seed"]))
    o.reset()
    assert np.array_equal(o.obs()[0], g["first_frame"])
    for t, acts in enumerate(g["actions"]):
        o.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), g["rewards"][t].view(np.uint32)), t
        assert np.array_equal(o.dones(), g["dones"][t]), t
    assert np.array_equal(o.state(0).view(np.uint32), g["final_state0"].view(np.uint32))
    assert np.array_equal(o.obs()[0], g["last_frame"])
    o.close()


def test_oracle_golden_scenarios(built):
    """every other scenario against tests/golden/scenarios_golden.npz: level dumps at reset, then rewards / dones over a fixed
    action stream and the final states (bit patterns)"""
    import helpers
    import orc

    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden

    g = np.load(os.path.join(ROOT, "tests", "golden", "scenarios_golden.npz"))
    for name in make_golden.SCENARIOS:
        levels, rewards, dones, states = make_golden.scenario_run(name)
        for e, lv in enumerate(levels):
            assert np.array_equal(lv, g["%s_level%d" % (name, e)]), "%s level %d" % (name, e)
        assert np.array_equal(rewards.view(np.uint32), g[name + "_rewards"].view(np.uint32)), name
        assert np.array_equal(dones, g[name + "_dones"]), name
        for e, st in enumerate(states):
            assert np.array_equal(st.view(np.uint32), g["%s_state%d" % (name, e)].view(np.uint32)), "%s state %d" % (name, e)


def test_mesh_tables_match_reference_magnum(built):
    """the oracle's mesh tables are the reference's Magnum primitives (counts from SURVEY.md 2.1) and the product's
    __constant__ tables hold the same bits"""
    import re
    import orc

    counts = {0: (24, 36), 1: (66, 384), 2: (42, 240), 3: (12, 36), 4: (26, 72)}
    names = {0: "box", 1: "capsule", 2: "sphere", 3: "cone", 4: "cylinder"}
    inc = open(os.path.join(ROOT, "megaverse_b200", "csrc", "mesh_tables.inc")).read()
    for t, (nv, ni) in counts.items():
        vtx, idx = orc.mesh(t)
        assert vtx.shape == (nv, 6) and idx.shape == (ni,)
        body = inc[inc.index("c_%sVerts" % names[t]):]
        body = body[: body.index("};")]
        vals = np.array([float.fromhex(x.rstrip("f")) for x in re.findall(r"-?0x[0-9a-f.]+p[+-]\d+f", body)], dtype=np.float32)
        assert np.array_equal(vals.view(np.uint32).reshape(nv, 6), vtx), names[t]
        ibody = inc[inc.index("c_%sIdx" % names[t]):]
        ibody = ibody[ibody.index("{") + 1: ibody.index("};")]
        assert np.array_equal(np.array([int(x) for x in ibody.replace("\n", " ").split(",") if x.strip()]), idx), names[t]
    # unit normals, box is the +-1 cube
    v, _ = orc.mesh(0)
    assert set(np.unique(v[:, :3].view(np.float32)).tolist()) == {-1.0, 1.0}
    for t in counts:
        v, _ = orc.mesh(t)
        nrm = np.linalg.norm(v[:, 3:].view(np.float32), axis=1)
        assert np.allclose(nrm, 1.0, atol=1e-5)


def test_analytic_sweep_agrees_with_its_definition(built):
    """The narrow phase that stands in for Bullet's convex sweep (oracle/orc_physics.hpp header) is DEFINED as: the first t in [0,1] at
    which the agent capsule penetrates the collider by allowedCcdPenetration (0.04); an already deeper start reports t = 0 only when
    moving into the surface.  Checked here against the independent signed-distance function (the one recoverFromPenetration uses) by
    dense sampling along random sweeps -- boxes axis-aligned and turned about Y, and other agents' capsules."""
    import ctypes as C

    import orc

    O = orc.lib()
    O.orc_sweep_case.argtypes = [C.c_void_p] * 5
    O.orc_capsule_distance.argtypes = [C.c_void_p] * 3
    O.orc_capsule_distance.restype = C.c_float
    rng = np.random.default_rng(12)
    n3 = np.zeros(3, np.float32)

    def dist(col, p):
        p = np.ascontiguousarray(p, np.float32)
        return float(O.orc_capsule_distance(col.ctypes.data, p.ctypes.data, n3.ctypes.data))

    hits = misses = starts_inside = 0
    for case in range(4000):
        kind = 0 if rng.random() < 0.8 else 1
        col = np.zeros(8, np.float32)
        col[0] = kind
        col[1:4] = rng.uniform(-2, 2, 3)
        col[4:7] = rng.uniform(0.05, 3.0, 3)
        col[7] = 0.0 if rng.random() < 0.5 else rng.uniform(-3.1, 3.1)
        a = rng.normal(size=3); a /= np.linalg.norm(a)
        reach = float(np.linalg.norm(col[4:7])) + 1.5
        f = (col[1:4] + a * rng.uniform(0.2, 1.3) * reach).astype(np.float32)
        to = (col[1:4] + rng.normal(size=3) * 0.6 * reach).astype(np.float32) if rng.random() < 0.7 else (f + rng.normal(size=3).astype(np.float32) * 0.3)
        f, to = np.ascontiguousarray(f, np.float32), np.ascontiguousarray(to, np.float32)
        t = np.zeros(1, np.float32)
        hit = O.orc_sweep_case(col.ctypes.data, f.ctypes.data, to.ctypes.data, t.ctypes.data, n3.ctypes.data)
        n_hit = n3.copy()
        d = (to - f).astype(np.float64)
        length = float(np.linalg.norm(d))
        tol = 2e-4 + 1e-5 * reach
        d0 = dist(col, f)
        ts = np.linspace(0.0, 1.0, 129)
        ds = np.array([dist(col, f + d * s) for s in ts])
        if hit:
            hits += 1
            th = float(t[0])
            assert 0.0 <= th <= 1.0
            assert abs(float(np.linalg.norm(n_hit)) - 1.0) < 1e-4, "hit normal is not unit length"
            if th == 0.0:  # started at or beyond the tolerance: must be moving into the surface
                starts_inside += 1
                assert d0 <= -0.04 + tol, (case, d0)
                assert float(np.dot(n_hit, d)) <= 1e-6 * max(length, 1.0), (case, "t = 0 while moving away")
            else:
                dh = dist(col, f + d * th)
                assert abs(dh + 0.04) < tol, (case, "distance at the hit", dh)
                assert (ds[ts < th - 1e-3] > -0.04 - tol).all(), (case, "deeper than the tolerance before the reported hit")
        else:
            misses += 1
            # never crosses the tolerance surface from outside
            crossing = (ds[:-1] > -0.04 + tol) & (ds[1:] < -0.04 - tol)
            assert not crossing.any(), (case, "crossed the tolerance surface without a hit", float(ds.min()))
    assert hits > 800 and misses > 800 and starts_inside > 5, (hits, misses, starts_inside)


@pytest.mark.parametrize("scenario,num_agents,params", [
    ("ObstaclesEasy", 2, {"obstaclesMinNumPlatforms": 3, "obstaclesMaxNumPlatforms": 5, "obstaclesMinGap": 2, "obstaclesMaxGap": 4, "obstaclesMinLava": 2, "obstaclesMaxLava": 6,
                          "obstaclesMinHeight": 1, "obstaclesMaxHeight": 4, "obstaclesNumAllowedMaxDifficulty": 2}),
    ("ObstaclesHard", 3, {"obstaclesMinNumPlatforms": 1, "obstaclesMaxNumPlatforms": 3, "episodeLengthSec": 20.0}),
    ("TowerBuilding", 8, {"episodeLengthSec": 10.0, "verticalLookLimitRad": 0.9}),
    ("Collect", 8, {"episodeLengthSec": 30.0}),
])
def test_level_generation_with_custom_parameters_matches_oracle(built, scenario, num_agents, params):
    """the same comparison under non-default float parameters (the reference's FloatParams dict of MegaverseEnv(..., params=...))"""
    import orc
    from megaverse_b200 import capi

    for seed in range(80, 95):
        o = orc.Oracle(scenario, 1, num_agents, params=params, render=False)
        o.seed_env(0, seed)
        for episode in range(2):
            o.reset()
            want = o.level(0)
            got = capi.generate_level(scenario, num_agents, seed, episode, params)
            n = len(want)
            assert np.array_equal(want, got[:n]), "%s seed %d episode %d: first diff at %s" % (scenario, seed, episode, np.nonzero(want != got[:n])[0][:5])
        o.close()


def test_drop_in_surface_covers_the_reference_bindings(built):
    """every name the reference's pybind module defines (src/libs/bindings/megaverse.cpp:267-292) exists on ours, and every public method /
    attribute of the reference's Python MegaverseEnv (megaverse/megaverse_env.py) exists on our MegaverseEnv.  Parsed from the reference
    sources, so it only runs where /root/reference is mounted."""
    import ast
    import importlib
    import os
    import re

    bind = "/root/reference/src/libs/bindings/megaverse.cpp"
    pyenv = "/root/reference/megaverse/megaverse_env.py"
    if not (os.path.exists(bind) and os.path.exists(pyenv)):
        pytest.skip("/root/reference absent")
    names = re.findall(r'\.def\("([a-z_]+)"', open(bind).read())
    assert len(names) >= 18
    m = importlib.import_module("megaverse_b200.extension.megaverse")
    for n in names:
        assert hasattr(m, n) or hasattr(m.MegaverseGym, n), "binding %s is missing" % n
    tree = ast.parse(open(pyenv).read())
    cls = [c for c in tree.body if isinstance(c, ast.ClassDef) and c.name == "MegaverseEnv"][0]
    methods = [f.name for f in cls.body if isinstance(f, ast.FunctionDef) and not f.name.startswith("_")]
    init = [f for f in cls.body if isinstance(f, ast.FunctionDef) and f.name == "__init__"][0]
    ctor_args = [a.arg for a in init.args.args]
    attrs = sorted({t.attr for n in ast.walk(init) if isinstance(n, ast.Assign) for t in n.targets
                    if isinstance(t, ast.Attribute) and isinstance(t.value, ast.Name) and t.value.id == "self"})
    import inspect

    from megaverse_b200.megaverse_env import MegaverseEnv

    for n in methods:
        assert callable(getattr(MegaverseEnv, n, None)), "MegaverseEnv.%s is missing" % n
    ours = list(inspect.signature(MegaverseEnv.__init__).parameters)
    assert ours[:len(ctor_args)] == ctor_args, (ours, ctor_args)
    src = inspect.getsource(MegaverseEnv)
    for a in attrs:
        assert re.search(r"self\.%s\b" % re.escape(a), src), "attribute %s is not set by our MegaverseEnv" % a


def test_levels_of_any_size_are_generated(built):
    """the reference's voxel grid and box merge have no capacity (component_voxel_grid.hpp:108-187): neither has the product.  A Collect
    landscape that decomposes into more static boxes than the engine's initial array (found by fuzzing; it used to be refused) is generated
    like any other and equals the oracle's; no level of any scenario is ever skipped"""
    import ctypes as C

    import orc
    from megaverse_b200 import capi

    L = capi.lib()
    L.mv_debug_count_unfit_levels.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    seed = 889027061
    o = orc.Oracle("Collect", 1, 2, render=False)
    o.seed_env(0, seed)
    o.reset()
    want = o.level(0)
    got = capi.generate_level("Collect", 2, seed, 0)
    assert want[0] > 768, "the case is meant to exceed the initial static-box capacity (%d boxes)" % want[0]
    assert np.array_equal(want, got[:len(want)])
    o.close()
    assert L.mv_debug_count_unfit_levels(b"Collect", 2, seed, 3, None, None, 0) == 0
    assert sum(L.mv_debug_count_unfit_levels(b"Collect", 2, s, 10, None, None, 0) for s in range(20000, 20100)) == 0
    for scen in (b"TowerBuilding", b"ObstaclesHard", b"Rearrange", b"HexExplore", b"HexMemory"):
        assert sum(L.mv_debug_count_unfit_levels(scen, 2, s, 5, None, None, 0) for s in range(20000, 20040)) == 0, scen
