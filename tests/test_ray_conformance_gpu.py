"""The CUDA ray kernel on constructed scenes (mv_debug_cast_rays: the engine's own launch over caller-built envs): every family of
ray_scenes.py equals the CPU restatement (tests/oracle_seg/orc_rays.cpp) bit for bit and the float64 reference (ray_ref.py) within the
bound of test_ray_conformance_cpu.py; every lane count (A * R from 1 to 2 048, so that each lane's rays k = 0..3 and partial warps run)
gives the same bits as casting alone; masked envs keep their rows; pixel-centre rays agree with the CUDA rasteriser's segmentation and
depth on mirrored and mesh scenes; one engine-level lockstep with A * R above 512."""
import numpy as np
import pytest

import ray_ref
import ray_scenes as scenes
from test_ray_conformance_cpu import T_BOUND, check_against_reference

pytestmark = pytest.mark.gpu


def _launch(group, mask=None, fill=None):
    """one launch over the scenes of `group` (same A, dirs and max_dist): (dist, tag) as [env][agent][R]"""
    from megaverse_b200 import capi

    E, A = len(group), len(group[0]["views"])
    S = max(1, max(len(s["rows"]) for s in group))
    rows = np.zeros((E, S, 18), dtype=np.float32)
    tags = np.zeros((E, S), dtype=np.int32)
    counts = np.zeros(E, dtype=np.int32)
    for e, s in enumerate(group):
        n = len(s["rows"])
        rows[e, :n], tags[e, :n], counts[e] = s["rows"], s["tags"], n
        rows[e, n:, 0] = 9.0  # rows beyond the count are not read
    views = np.stack([s["views"] for s in group])
    R = len(group[0]["dirs"])
    dist, tag = (None, None) if fill is None else fill
    dist, tag = capi.cast_rays(views, rows, tags, counts, group[0]["dirs"], group[0]["max_dist"], mask, dist, tag)
    return dist.reshape(E, A, R), tag.reshape(E, A, R)


def _groups(fam):
    out = {}
    for s in fam:
        out.setdefault((len(s["views"]), s["dirs"].tobytes(), s["max_dist"]), []).append(s)
    return list(out.values())


def _same(where, got, want):
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), "%s: distance differs on %d rays" % (where, int((got[0] != want[0]).sum()))
    assert np.array_equal(got[1], want[1]), "%s: tag differs on %d rays" % (where, int((got[1] != want[1]).sum()))


@pytest.mark.parametrize("family", sorted(scenes.FAMILIES) + ["edges"])
def test_kernel_equals_the_restatement_and_the_reference(family):
    import orc_rays

    fam = scenes.edge_scenes(poses=20) + scenes.edge_scenes(poses=20, seed=1, far=True) if family == "edges" else scenes.FAMILIES[family]()
    for group in _groups(fam):
        dist, tag = _launch(group)
        for e, s in enumerate(group):
            for a in range(len(s["views"])):
                want = orc_rays.rays_scene(s["views"][a], s["rows"], s["tags"], s["dirs"], s["max_dist"], a)
                _same("%s env %d agent %d" % (family, e, a), (dist[e, a], tag[e, a]), want)
                if family == "edges":
                    assert (tag[e, a] != 0).all(), "a ray at a shared edge or vertex slips through"
                    continue
                res = ray_ref.cast(s["views"][a], s["rows"], s["tags"], s["dirs"], s["max_dist"], a)
                check_against_reference(family, dist[e, a], tag[e, a], res, s, a)


# A * R: one ray, partial warps either side of 32, 512 (one ray per lane), 513 (a second ray in one lane), 1 024, 1 533 / 1 536 (three
# rays per lane, the last warp partial) and 2 048 (four)
SHAPES = [(1, 1), (1, 31), (1, 33), (3, 11), (2, 256), (3, 171), (4, 256), (7, 219), (6, 256), (8, 256)]


@pytest.mark.parametrize("A,R", SHAPES)
def test_every_lane_count_gives_the_bits_of_casting_alone(A, R):
    """a launch of E envs x A agents x R rays equals the restatement for every ray, and every ray equals the same ray cast alone in a
    launch of one agent and at most 32 rays (lane k = 0 only)"""
    import orc_rays

    rng = np.random.default_rng(A * 1000 + R)
    base = scenes.meshes(seed=3)[:6] + scenes.boxes(seed=3)[8:14]
    group = []
    dirs = np.concatenate([scenes.grid_dirs(16, 0.35), scenes.grid_dirs(16, 0.2)])[rng.permutation(512)[:R]]
    for s in base:
        views = [s["views"][0]] + [scenes._camera(rng)[0] for _ in range(A - 1)]
        group.append(scenes._scene(views, s["rows"], s["tags"], dirs))
    dist, tag = _launch(group)
    hits = 0
    for e, s in enumerate(group):
        for a in range(A):
            want = orc_rays.rays_scene(s["views"][a], s["rows"], s["tags"], dirs, s["max_dist"], a)
            _same("A=%d R=%d env %d agent %d" % (A, R, e, a), (dist[e, a], tag[e, a]), want)
            hits += int((tag[e, a] != 0).sum())
    assert hits > 0
    # alone: one env, agent a as the only agent, 32 rays at a time
    for e in (0, len(group) - 1):
        s = group[e]
        for a in {0, A - 1}:
            for k in range(0, R, 32):
                one = scenes._scene([s["views"][a]], s["rows"], s["tags"], dirs[k:k + 32])  # (no agent-tagged rows in these scenes)
                d1, t1 = _launch([one])
                _same("alone env %d agent %d rays %d.." % (e, a, k), (d1[0, 0], t1[0, 0]), (dist[e, a, k:k + 32], tag[e, a, k:k + 32]))


def test_masked_envs_keep_their_rows():
    fam = scenes.meshes(seed=7)[:9]
    E, R = len(fam), 256
    mask = (np.arange(E) % 3 != 1).astype(np.uint8)
    fill = (np.full((E, R), -7.5, dtype=np.float32), np.full((E, R), 0xBEEF, dtype=np.uint16))
    dist, tag = _launch(fam, mask, fill)
    full = _launch(fam)
    for e in range(E):
        if mask[e]:
            _same("env %d" % e, (dist[e, 0], tag[e, 0]), (full[0][e, 0], full[1][e, 0]))
        else:
            assert (dist[e, 0] == -7.5).all() and (tag[e, 0] == 0xBEEF).all(), "env %d was cast" % e
    assert (full[1][mask == 0] != 0).any()


# ---------------------------------------------------------------------------------------------------- against the CUDA rasteriser
def _mesh_scene(W, H, seed=0):
    """every mesh type at random poses and scales ahead of the camera, boxes first (draw order by mesh type)"""
    import raster_scenes as rsc

    rng = np.random.default_rng(seed)
    rows = []
    for k in range(14):
        z = rng.uniform(3.0, 12.0)
        x, y = rsc._view_xy(rng.uniform(0.1, 0.9) * W, rng.uniform(0.1, 0.9) * H, z, W, H)
        rows.append(rsc._row(k % 5, k, rsc._model([x, y, -z], rng.uniform(0.3, 1.2, 3), rsc._rot(*rng.uniform(0, 2 * np.pi, 3)))))
    return rsc._scene(rows)


@pytest.mark.parametrize("family", ["mirrored", "meshes"])
def test_pixel_centre_rays_agree_with_the_cuda_rasteriser(family):
    import raster_ref
    import raster_scenes as rsc
    from megaverse_b200 import capi

    W, H = 128, 72
    view16, inst = rsc.mirrored(W, H) if family == "mirrored" else _mesh_scene(W, H)
    _, depth, seg = capi.render_instances(view16, inst, W, H, want_depth=True, segmentation=True, fast=0)
    p00, p11, _, _ = raster_ref.projection(W, H)
    px, py = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    nx, ny = (px + 0.5 - W / 2) / (W / 2), (py + 0.5 - H / 2) / (H / 2)
    dirs = np.stack([nx / float(p00), ny / float(p11), -np.ones_like(nx)], -1).reshape(-1, 3).astype(np.float32)
    n = len(inst)
    tags = np.arange(1, n + 1, dtype=np.int32)
    dist = np.zeros(W * H, dtype=np.float32)
    tag = np.zeros(W * H, dtype=np.uint16)
    for k in range(0, W * H, 256):
        d, t = capi.cast_rays(view16.reshape(1, 1, 16), inst.reshape(1, n, 18), tags.reshape(1, n), [n], dirs[k:k + 256], 120.0)
        dist[k:k + 256], tag[k:k + 256] = d[0], t[0]
    dist, tag = dist.reshape(H, W), tag.reshape(H, W)
    ok = (tag == seg) & (np.abs(dist - depth) <= 0.01 * np.maximum(depth, 1e-30))
    # away from silhouettes: the 5 x 5 neighbourhood shows one drawable (or none)
    pad = np.pad(seg.astype(np.int32), 2, mode="edge")
    interior = np.ones_like(seg, dtype=bool)
    for dy in range(5):
        for dx in range(5):
            interior &= pad[dy:dy + H, dx:dx + W] == seg
    assert interior.sum() > W * H // 2 and (seg[interior] != 0).sum() > 300
    assert ok[interior].all(), "%s: %d interior pixels disagree" % (family, int((~ok[interior]).sum()))
    assert ok.mean() >= 0.995, "%s: %.4f of pixels agree" % (family, ok.mean())
    if family == "mirrored":
        mirrored_rows = [i for i in range(n) if np.linalg.det(inst[i, 2:].reshape(4, 4)[:3, :3].astype(np.float64)) < 0]
        assert np.isin(seg[interior], np.array(mirrored_rows) + 1).sum() > 200, "mirrored instances cover interior pixels"


# ---------------------------------------------------------------------------------------------------- engine lockstep with A * R > 512
def test_engine_lockstep_with_two_rays_per_lane():
    """Collect 2 x 4 at R = 256 (A * R = 1 024: two rays per lane) for 20 steps against the restatement on the oracle's scenes"""
    import helpers
    import orc
    import orc_rays
    from megaverse_b200 import capi, rays
    from test_cameras_gpu import _params

    E, A, seed, maxd = 2, 4, 1000, 60.0
    dirs = rays.fan(256, 360.0)
    o = orc.Oracle("Collect", E, A, render=False, params=_params("Collect"))
    g = capi.Engine("Collect", E, A, 128, 72, num_threads=2, params=_params("Collect"))
    g.set_rays(dirs, maxd)
    try:
        for e in range(E):
            o.seed_env(e, seed + 7919 * e)
            g.seed_env(e, seed + 7919 * e)
        o.reset()
        g.reset()
        rng = np.random.default_rng(4)
        for t in range(20):
            acts = helpers.purposeful_actions(rng, E * A, t)
            o.step(acts)
            g.step(acts)
            d, tg = g.rays()
            _same("step %d" % t, (np.array(d), np.array(tg)), orc_rays.rays_all(o, dirs, maxd))
    finally:
        o.close()
        g.close()
