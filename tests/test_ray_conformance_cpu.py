"""Ray sensors without a GPU: the CPU restatement of the hit definition (tests/oracle_seg/orc_rays.cpp, which the kernel equals bit for bit)
against an independent float64 reference (ray_ref.py) on the constructed scene families of ray_scenes.py, each of which first proves
that it reached its case.  Plus the two properties the definition's handling of mirrored models and mesh edges establishes, and the
argument checks of the debug entry mv_debug_cast_rays (they run before any device call).

Where every margin of a ray clears ray_ref.Result.robust's thresholds, the tag must match and t must agree within
T_BOUND * 2^-24 * cond(model) relative, cond the 2-norm condition number of the winning row's 3 x 3 part.  Measured maximum of
|t - t_ref| / (t_ref * 2^-24 * cond) over the families: 169 (mirrored; boxes 11, meshes 46), so the bound is 512."""
import numpy as np
import pytest

import ray_ref
import ray_scenes as scenes

T_BOUND = 512.0
EPS32 = 2.0 ** -24


def check_against_reference(family, dist, tag, res, scene, agent):
    """the tag where the reference is robust (everywhere for the exact families) and t within the bound"""
    rob = res.robust()
    exact = family in ("ties", "zero_components", "inside_and_on", "singular", "max_distance", "own_drawables")
    if exact:  # exact constructions: every decision is exact in float32 as in float64, ties and borders included
        rob = np.ones_like(rob)
    bad = np.nonzero(tag[rob] != res.tag[rob])[0]
    assert bad.size == 0, "%s: tag differs on %d robust rays (first: ray %d, %d against %d)" % (
        family, bad.size, np.nonzero(rob)[0][bad[0]], tag[rob][bad[0]], res.tag[rob][bad[0]])
    h = rob & (res.tag != 0)
    rel = np.abs(dist[h].astype(np.float64) - res.dist[h]) / res.dist[h] / (EPS32 * res.cond[h])
    assert rel.max(initial=0.0) <= T_BOUND, "%s: t differs by %.1f x 2^-24 x cond" % (family, rel.max())
    assert (dist[~rob & (tag == 0)] == 0).all()
    return int(rob.sum()), float(rel.max(initial=0.0))


@pytest.mark.parametrize("family", sorted(scenes.FAMILIES))
def test_restatement_against_the_float64_reference(family):
    import orc_rays

    fam = scenes.FAMILIES[family]()
    results, checked, rays = [], 0, 0
    for s in fam:
        rs = []
        for a in range(len(s["views"])):
            res = ray_ref.cast(s["views"][a], s["rows"], s["tags"], s["dirs"], s["max_dist"], a)
            dist, tag = orc_rays.rays_scene(s["views"][a], s["rows"], s["tags"], s["dirs"], s["max_dist"], a)
            n, _ = check_against_reference(family, dist, tag, res, s, a)
            checked += n
            rays += tag.size
            rs.append(res)
        results.append(rs)
    scenes.check_reach(family, fam, results)
    assert checked >= 0.6 * rays, "%s: only %d of %d rays are far enough from every decision to be checked" % (family, checked, rays)


def test_mirrored_instances_show_their_far_faces():
    """the rasteriser draws a mirrored instance from its far faces (its winding turns round on screen), so the rays see those: a box
    of half extent 1 at z = -5 is met at its back face, t = 6, under every mirror; two negative scales are a rotation and show the front"""
    import orc_rays

    for sign in scenes.SIGNS + [(1, 1, 1)]:
        row = scenes._row(0, scenes._model([0, 0, -5.0], sign))
        dist, tag = orc_rays.rays_scene(scenes.EYE, row[None], [1], [[0, 0, -1]], 100.0)
        want = 6.0 if np.prod(sign) < 0 else 4.0
        assert dist[0] == want and tag[0] == 1, (sign, dist[0])
    # meshes: the far side, as the reference finds it
    for kind in range(1, 5):
        for sign in scenes.SIGNS:
            row = scenes._row(kind, scenes._model([0, 0, -5.0], sign))
            dist, _ = orc_rays.rays_scene(scenes.EYE, row[None], [1], [[0, 0, -1], [0.05, 0.02, -1]], 100.0)
            res = ray_ref.cast(scenes.EYE, row[None], [1], [[0, 0, -1], [0.05, 0.02, -1]], 100.0)
            assert np.allclose(dist, res.dist, rtol=1e-5) and ((dist > 5.0) == (np.prod(sign) < 0)).all(), (kind, sign, dist)


def test_rays_at_shared_edges_and_vertices_hit():
    """every ray aimed at an edge or a vertex where front faces (facing margin >= 0.2) of a mesh meet hits the mesh, under 20 poses per
    mesh type, near and far (origins up to thousands of object units away); without the widened bounds 38 capsule, 49 sphere and 5
    cylinder rays of the near poses slip through.  Rays through the faces' centroids keep the reference's t."""
    import orc_rays

    per_kind = {}
    for s in scenes.edge_scenes(poses=20) + scenes.edge_scenes(poses=20, seed=1, far=True):
        kind = int(s["rows"][0, 0])
        dist, tag = orc_rays.rays_scene(s["views"][0], s["rows"], s["tags"], s["dirs"], s["max_dist"], 0)
        miss = int((tag == 0).sum())
        assert miss == 0, "mesh %d: %d of %d rays at shared edges and vertices miss" % (kind, miss, tag.size)
        per_kind[kind] = per_kind.get(kind, 0) + tag.size
        res = ray_ref.cast(s["views"][0], s["rows"], s["tags"], s["dirs"], s["max_dist"], 0)
        assert (res.tag != 0).all()
        assert np.allclose(dist, res.dist, rtol=1e-4)
    assert sorted(per_kind) == [1, 2, 3, 4] and min(per_kind.values()) >= 40, per_kind
    rng = np.random.default_rng(5)
    for kind in range(1, 5):
        P, I = ray_ref.mesh(kind)
        view, C = scenes._camera(rng)
        row = scenes._row(kind, scenes._model((C @ np.array([0, 0, -6.0, 1.0]))[:3], [1.0, 1.3, 0.8], C[:3, :3] @ scenes._rot(rng)))
        M = row[2:].astype(np.float64).reshape(4, 4).T
        W = P @ M[:3, :3].T + M[:3, 3]
        n = np.cross(W[I[:, 1]] - W[I[:, 0]], W[I[:, 2]] - W[I[:, 0]])
        cen = W[I].mean(axis=1)
        d = cen - C[:3, 3]
        front = -(n * d).sum(1) >= 0.2 * np.linalg.norm(n, axis=1) * np.linalg.norm(d, axis=1)
        Cinv = np.linalg.inv(C)
        dirs = (cen[front] @ Cinv[:3, :3].T + Cinv[:3, 3])[:256]
        assert len(dirs) >= 4
        dist, tag = orc_rays.rays_scene(view, row[None], [1], dirs, 100.0)
        res = ray_ref.cast(view, row[None], [1], dirs, 100.0)
        assert (tag == 1).all() and (res.tag == 1).all()
        rel = np.abs(dist - res.dist) / res.dist / (EPS32 * res.cond)
        assert rel.max() <= T_BOUND


def test_debug_cast_refuses_bad_arguments(built):
    """mv_debug_cast_rays checks every pointer and range before it touches the device"""
    import ctypes as C
    from megaverse_b200 import capi

    L = capi.lib()
    E, A, S, R = 2, 2, 4, 8
    views = np.tile(scenes.EYE, (E * A, 1)).astype(np.float32)
    rows = np.zeros((E, S, 18), dtype=np.float32)
    rows[:, :, 2:] = scenes.EYE
    tags = np.zeros((E, S), dtype=np.int32)
    counts = np.array([S, 1], dtype=np.int32)
    dirs = scenes.grid_dirs(2, 0.1)[:R].copy()
    dist = np.zeros((E * A, R), dtype=np.float32)
    tag = np.zeros((E * A, R), dtype=np.uint16)
    ptr = lambda a: a.ctypes.data

    def call(views=views, rows=rows, tags=tags, counts=counts, E=E, A=A, S=S, dirs=dirs, R=R, maxd=10.0, dist=dist, tag=tag):
        return L.mv_debug_cast_rays(views if views is None else ptr(views), rows if rows is None else ptr(rows), tags if tags is None else ptr(tags),
                                    counts if counts is None else ptr(counts), E, A, S, dirs if dirs is None else ptr(dirs), R, C.c_float(maxd), None,
                                    dist if dist is None else ptr(dist), tag if tag is None else ptr(tag))

    for kw in ({"views": None}, {"rows": None}, {"tags": None}, {"counts": None}, {"dirs": None}, {"dist": None}, {"tag": None}):
        assert call(**kw) == capi.MV_ERR_ARG, kw
    for kw in ({"E": 0}, {"A": 0}, {"A": 9}, {"R": 0}, {"R": 257}, {"S": 0}, {"S": 65537}, {"maxd": 0.0}, {"maxd": -1.0}, {"maxd": float("inf")},
               {"maxd": float("nan")}):
        assert call(**kw) == capi.MV_ERR_ARG, kw
    for c in ([S + 1, 0], [-1, 0]):
        assert call(counts=np.array(c, dtype=np.int32)) == capi.MV_ERR_ARG, c
    for m in (5.0, -1.0, 1.5, float("nan")):
        bad = rows.copy()
        bad[1, 0, 0] = m  # env 1 casts only row 0
        assert call(rows=bad) == capi.MV_ERR_ARG, m
    assert callable(capi.cast_rays) and "mv_debug_cast_rays" in capi.EXPORTS
