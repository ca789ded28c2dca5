"""An INDEPENDENT restatement of the fixed-function rasterisation rules against the oracle's rasteriser (CPU only).

The reference draws with Vulkan (V4R: vulkan_state.cpp:588-606 -- back-face culling with counter-clockwise fronts, depth test
LESS_OR_EQUAL on a D32 attachment, one sample per pixel) and its tests hold no pixel vector, so the oracle's triangle rasteriser
(oracle/orc_raster.hpp) could so far only be compared with itself.  The rules it restates are not reference code but the Vulkan
specification's: view-volume clipping 0 <= z_c <= w_c, the viewport transform, fixed-point vertex positions (8 sub-pixel bits),
one sample at the pixel centre, the top-left rule for samples exactly on an edge, depth interpolated linearly in window space,
perspective-correct interpolation of the varyings (here: clip-space w, which V4R writes out as its depth image).

raster_ref.py implements those rules a second time, in a different form and in different arithmetic (exact integer coverage with an
infinitesimal-displacement tie rule, float64 depth and w, float64 Sutherland-Hodgman clipping, unbounded window coordinates); this file
checks it against the oracle, on random scenes here and on every constructed scene family of test_raster_conformance_gpu.py, and
bounds the window coordinates the product's own scenes produce (the envelope inside which the kernel's integer set-up is exact).

Compared: the oracle's depth image (view-space w of the visible fragment, 0 = nothing drawn) -- its zero pattern IS the coverage
mask.  Scenes without clipping must agree in every pixel (coverage exactly, depth to float32 rounding); scenes cut by the near
plane (the clipper creates new vertices, whose float32 vs float64 positions can snap one sub-pixel apart) in all but a handful.
Colour: raster_ref.shade64 restates the fragment stage (uber.frag:112-141) in float64 on float64 varyings (camera-space position and
normal, the normal by numpy's inverse transpose, carried through the clipper, interpolated with perspective correction); the oracle's
float32 bytes must follow raster_ref.colour_rule, whose tolerance is derived there.
"""
import warnings

import numpy as np
import pytest

import orc
import raster_ref as ref

W, H = 128, 72
F32 = np.float32


def _projection():
    return ref.projection(W, H)


STATS = {"ties": 0}  # samples that lay exactly on an edge of a front-facing triangle (the cases the tie rule decides)


def _independent_depth(view16, instances):
    """depth image (view-space w of the visible fragment, 0 = empty) by the rules of the specification at 128 x 72; also returns whether
    any primitive needed clipping"""
    R = ref.render(view16, instances, W, H)
    STATS["ties"] += R.ties
    return R.w, R.clipped


def _random_scene(rng, n, near_camera):
    """instances (mesh, colour, model matrix column-major) in front of a camera at the origin looking down -z with a random roll"""
    rows = []
    for _ in range(n):
        mesh = int(rng.choice([0, 0, 0, 1, 2, 3, 4]))
        s = rng.uniform(0.2, 1.5, size=3) * (3.0 if near_camera and mesh == 0 and rng.random() < 0.3 else 1.0)
        ang = rng.uniform(0, 2 * np.pi, size=3)
        cx, sx_ = np.cos(ang[0]), np.sin(ang[0]); cy, sy_ = np.cos(ang[1]), np.sin(ang[1]); cz, sz_ = np.cos(ang[2]), np.sin(ang[2])
        rx = np.array([[1, 0, 0], [0, cx, -sx_], [0, sx_, cx]]); ry = np.array([[cy, 0, sy_], [0, 1, 0], [-sy_, 0, cy]]); rz = np.array([[cz, -sz_, 0], [sz_, cz, 0], [0, 0, 1]])
        rot = rz @ ry @ rx @ np.diag(s)
        depth = rng.uniform(0.3, 3.0) if near_camera else rng.uniform(4.0, 14.0)
        t = np.array([rng.uniform(-1.2, 1.2) * depth, rng.uniform(-0.8, 0.8) * depth, -depth])
        m = np.eye(4); m[:3, :3] = rot; m[:3, 3] = t
        rows.append(np.concatenate([[mesh, rng.integers(0, 20)], m.T.reshape(-1)]))  # column-major
    rows.sort(key=lambda r: r[0])  # draw order: by mesh type, boxes first (what the product's instance lists guarantee)
    roll = rng.uniform(-0.3, 0.3)
    v = np.eye(4); v[:2, :2] = [[np.cos(roll), -np.sin(roll)], [np.sin(roll), np.cos(roll)]]
    return v.T.reshape(-1).astype(F32), np.array(rows, dtype=F32)


def _compare(view16, inst):
    _, ref = orc.render_instances(view16, inst, W, H, want_depth=True)
    mine, clipped = _independent_depth(view16, inst)
    cov_ref, cov_mine = ref > 0, mine > 0
    both = cov_ref & cov_mine
    rel = np.abs(ref[both].astype(np.float64) - mine[both]) / mine[both] if both.any() else np.zeros(0)
    return cov_ref, cov_mine, rel, clipped


def _colour(view16, inst, W, H, R=None):
    """the oracle's colour against the float64 fragment stage (raster_ref.colour_rule) where both draw the same surface (depth within
    2e-5): (broken bytes, differing bytes, worst margin among them, largest difference)"""
    R = ref.render(view16, inst, W, H) if R is None else R
    rgba, od = orc.render_instances(view16, inst, W, H, want_depth=True)
    same = (od > 0) & (R.w > 0)
    same[same] = np.abs(od[same].astype(np.float64) - R.w[same]) / R.w[same] < 2e-5
    return ref.colour_rule(R.frag, rgba, same)


@pytest.mark.parametrize("seed", range(8))
def test_unclipped_scenes_agree_in_every_pixel(seed):
    rng = np.random.default_rng(1000 + seed)
    view16, inst = _random_scene(rng, 6, near_camera=False)
    cov_ref, cov_mine, rel, clipped = _compare(view16, inst)
    assert not clipped
    assert cov_ref.sum() > 50, "the scene should cover some pixels"
    assert np.array_equal(cov_ref, cov_mine), "coverage differs in %d pixels" % int((cov_ref != cov_mine).sum())
    # same visible surface: w agrees to float32 rounding of the oracle's arithmetic (a different winner would be a different surface)
    assert rel.max() < 2e-5, "depth differs by %.3g" % rel.max()
    broken, differ, worst, dmax = _colour(view16, inst, W, H)
    assert broken == 0, "%d colour bytes break the rule (%d differ, by up to %d)" % (broken, differ, dmax)


@pytest.mark.parametrize("seed", range(6))
def test_scenes_cut_by_the_near_plane_agree(seed):
    rng = np.random.default_rng(2000 + seed)
    view16, inst = _random_scene(rng, 5, near_camera=True)
    cov_ref, cov_mine, rel, _ = _compare(view16, inst)
    assert cov_ref.sum() > 200
    mism = int((cov_ref != cov_mine).sum())
    assert mism <= 8, "coverage differs in %d pixels" % mism  # new vertices made by the clipper may snap one sub-pixel apart
    assert (rel > 1e-4).sum() <= 8, "visible surface differs in %d pixels" % int((rel > 1e-4).sum())
    broken, differ, worst, dmax = _colour(view16, inst, W, H)
    assert broken <= 3 * 8, "%d colour bytes break the rule (%d differ, by up to %d)" % (broken, differ, dmax)


@pytest.mark.parametrize("seed", range(4))
def test_edges_through_pixel_centres(seed):
    """random scenes almost never put a sample exactly on an edge, so the tie rule needs scenes built for it: boxes facing the camera whose
    front-face corners project onto pixel centres (within the 1/512-pixel reach of the fixed-point snap) -- whole rows and columns of
    samples, and the diagonal the face's two triangles share, lie exactly on edges.  Coverage must still agree in every pixel."""
    rng = np.random.default_rng(3000 + seed)
    p00, p11, _, _ = _projection()
    rows = []
    for k in range(5):
        z_front = -rng.uniform(3.0, 9.0)
        half_z = rng.uniform(0.2, 0.6)
        px0, py0 = int(rng.integers(4, 90)), int(rng.integers(4, 50))
        wpx = int(rng.integers(6, 30)); hpx = wpx if k % 2 == 0 else int(rng.integers(6, 20))  # squares: the shared diagonal hits pixel centres too
        x0, x1 = [((px + 0.5) - W / 2) / (W / 2) * (-z_front) / float(p00) for px in (px0, px0 + wpx)]
        y0, y1 = [((py + 0.5) - H / 2) / (H / 2) * (-z_front) / float(p11) for py in (py0, py0 + hpx)]
        m = np.eye(4)
        m[0, 0], m[1, 1], m[2, 2] = abs(x1 - x0) / 2, abs(y1 - y0) / 2, half_z
        m[:3, 3] = [(x0 + x1) / 2, (y0 + y1) / 2, z_front - half_z]
        rows.append(np.concatenate([[0, k], m.T.reshape(-1)]))
    view16 = np.eye(4, dtype=F32).reshape(-1)
    inst = np.array(rows, dtype=F32)
    STATS["ties"] = 0
    cov_ref, cov_mine, rel, clipped = _compare(view16, inst)
    assert not clipped
    assert STATS["ties"] > 100, "the scene was built to put samples on edges (%d)" % STATS["ties"]
    assert np.array_equal(cov_ref, cov_mine), "coverage differs in %d pixels" % int((cov_ref != cov_mine).sum())
    assert rel.max() < 2e-5


def test_shared_edges_are_drawn_exactly_once():
    """the tie rule's purpose: two triangles sharing an edge cover every sample on it exactly once -- a fan of thin triangles around a
    vertex placed exactly on a pixel centre, edges through many pixel centres; checked on the independent rule itself and through the
    oracle (a full-screen quad of two triangles plus axis-aligned boxes whose edges run through pixel centres leave no hole)"""
    cx, cy = 64 * 256 + 128, 36 * 256 + 128
    ys, xs = np.mgrid[0:H, 0:W]
    sx = (xs * 256 + 128).astype(np.int64); sy = (ys * 256 + 128).astype(np.int64)
    ring = [(cx + int(30 * 256 * np.cos(a)) // 128 * 128, cy + int(30 * 256 * np.sin(a)) // 128 * 128) for a in np.linspace(0, 2 * np.pi, 17)[:-1]]
    count = np.zeros((H, W), dtype=int)
    for k in range(16):
        (x1, y1), (x2, y2) = ring[k], ring[(k + 1) % 16]
        tri = [(cx, cy), (x2, y2), (x1, y1)]
        area2 = (tri[1][0] - tri[0][0]) * (tri[2][1] - tri[0][1]) - (tri[1][1] - tri[0][1]) * (tri[2][0] - tri[0][0])
        if area2 > 0:
            tri = [tri[0], tri[2], tri[1]]
        inside = np.ones((H, W), dtype=bool)
        for (ax, ay), (bx, by) in ((tri[1], tri[2]), (tri[2], tri[0]), (tri[0], tri[1])):
            dEdx, dEdy = (by - ay), -(bx - ax)
            E = dEdx * (sx - ax) + dEdy * (sy - ay)
            inside &= (E > 0) | ((E == 0) & (dEdx > 0 or (dEdx == 0 and dEdy > 0)))
        count += inside
    assert count.max() == 1, "a sample was covered twice"
    assert count[36, 64] == 1, "the shared vertex on a pixel centre belongs to exactly one triangle"
    interior = (sx - cx) ** 2 + (sy - cy) ** 2 < (25 * 256) ** 2
    assert (count[interior] == 1).all(), "a sample inside the fan was not covered"


def _tie_scene(seed):
    rng = np.random.default_rng(3000 + seed)
    p00, p11, _, _ = _projection()
    rows = []
    for k in range(5):
        z_front = -rng.uniform(3.0, 9.0)
        half_z = rng.uniform(0.2, 0.6)
        px0, py0 = int(rng.integers(4, 90)), int(rng.integers(4, 50))
        wpx = int(rng.integers(6, 30)); hpx = wpx if k % 2 == 0 else int(rng.integers(6, 20))
        x0, x1 = [((px + 0.5) - W / 2) / (W / 2) * (-z_front) / float(p00) for px in (px0, px0 + wpx)]
        y0, y1 = [((py + 0.5) - H / 2) / (H / 2) * (-z_front) / float(p11) for py in (py0, py0 + hpx)]
        m = np.eye(4)
        m[0, 0], m[1, 1], m[2, 2] = abs(x1 - x0) / 2, abs(y1 - y0) / 2, half_z
        m[:3, 3] = [(x0 + x1) / 2, (y0 + y1) / 2, z_front - half_z]
        rows.append(np.concatenate([[0, k], m.T.reshape(-1)]))
    return np.eye(4, dtype=F32).reshape(-1), np.array(rows, dtype=F32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,seed", [("far", 0), ("far", 1), ("ties", 0), ("ties", 1), ("near", 0)])
def test_cuda_rasteriser_against_the_independent_rules(kind, seed):
    """the CUDA kernel itself (mv_debug_render_instances: the product's viewKernel on one view) against this file's restatement of the
    specification -- no oracle in between"""
    from megaverse_b200 import capi

    if kind == "ties":
        view16, inst = _tie_scene(seed)
    else:
        rng = np.random.default_rng((1000 if kind == "far" else 2000) + seed)
        view16, inst = _random_scene(rng, 6 if kind == "far" else 5, near_camera=(kind == "near"))
    _, dev = capi.render_instances(view16, inst, W, H, want_depth=True)
    mine, _ = _independent_depth(view16, inst)
    cov_dev, cov_mine = dev > 0, mine > 0
    mism = int((cov_dev != cov_mine).sum())
    assert mism <= (8 if kind == "near" else 0), "coverage differs in %d pixels" % mism
    both = cov_dev & cov_mine
    rel = np.abs(dev[both].astype(np.float64) - mine[both]) / mine[both]
    assert (rel > (1e-4 if kind == "near" else 2e-5)).sum() <= (8 if kind == "near" else 0)


# ---------------------------------------------------------------------------------------------------- constructed scene families
import raster_scenes as scenes  # noqa: E402


@pytest.mark.parametrize("size", [(128, 72), (64, 64), (32, 512), (512, 32), (160, 96)])
@pytest.mark.parametrize("family", sorted(scenes.FAMILIES))
def test_scene_families_reach_their_branch_and_agree_with_the_oracle(family, size):
    """every constructed family of test_raster_conformance_gpu.py, drawn by the restatement: it reaches what it was built for, and the
    oracle agrees with it as on the random scenes (the window coordinates stay far inside the int32 range the oracle snaps to) -- in
    coverage, depth and colour (raster_ref.colour_rule: within 1 LSB of the float64 fragment stage, and different only within M LSB of
    a rounding boundary; clipped families and sizes other than 128 x 72 in at most 8 pixels' worth of bytes, where near-equal depths of
    two surfaces or clipper vertices one sub-pixel apart make the two sides draw different surfaces)"""
    W, H = size
    view16, inst = scenes.build(family, W, H)
    R = ref.render(view16, inst, W, H)
    scenes.check_reach(family, R, W, H)
    assert max(t["max_coord"] for t in R.tris) < (1 << 30)
    _, od = orc.render_instances(view16, inst, W, H, want_depth=True)
    cov_ref, cov_mine = od > 0, R.w > 0
    mism = int((cov_ref != cov_mine).sum())
    both = cov_ref & cov_mine
    rel = np.abs(od[both].astype(np.float64) - R.w[both]) / R.w[both]
    if family in scenes.CLIPPED:
        assert mism <= 8 and (rel > 1e-4).sum() <= 8, "coverage differs in %d pixels" % mism
    else:
        assert mism == 0, "coverage differs in %d pixels" % mism
        assert rel.max() < 1e-4 and (rel > 2e-5).sum() <= (0 if size == (128, 72) else 8), "depth differs by %.3g" % rel.max()
    broken, differ, worst, dmax = _colour(view16, inst, W, H, R)
    print("%s %dx%d: %d colour bytes differ from the float64 ones (by up to %d), worst boundary margin among them %.4f LSB" % (
        family, W, H, differ, dmax, worst))
    loose = 0 if size == (128, 72) and family not in scenes.CLIPPED else 3 * 8
    assert broken <= loose, "%d colour bytes break the rule (%d differ, by up to %d)" % (broken, differ, dmax)


def test_reference_takes_window_coordinates_unbounded():
    """a vertex 2^24 pixels off-screen, just in front of the near plane: the restatement keeps its snapped coordinate exact (no int32
    saturation or wrap) and still draws the on-screen part of the triangle, which covers the samples a guard-band rasteriser covers"""
    view16, inst = scenes.offscreen_vertex(128, 72, 24, opposite=False)
    R = ref.render(view16, inst, 128, 72)
    assert max(t["max_coord"] for t in R.tris) > (1 << 31)
    assert (R.w > 0).sum() > 100


# ---------------------------------------------------------------------------------------------------- the window-coordinate envelope
SCENARIOS = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]


def _window_extent(view16, inst):
    """largest |x_ndc|, |y_ndc| and largest difference of x_ndc, y_ndc between two corners of a triangle, over every vertex a rasteriser sets
    up for this view at 128 x 72 (inside both planes, or made by the near / far clip), excluding triangles wholly beyond one side plane"""
    ext = np.zeros(4)
    for mesh_kind in np.unique(inst[:, 0]).astype(int):
        rows = inst[inst[:, 0] == mesh_kind]
        verts, tris = ref.mesh(mesh_kind)
        for row in rows:
            c = ref.vertex_stage(view16, row[2:18], verts, W, H).astype(np.float64)[tris]   # [t][3][4]
            d_near, d_far = c[..., 2], c[..., 3] - c[..., 2]
            pts, ok = [c], [(d_near >= 0) & (d_far >= 0)]
            for d, other in ((d_near, d_far), (d_far, d_near)):
                for a, b in ((0, 1), (1, 2), (2, 0)):
                    cross = (d[:, a] >= 0) != (d[:, b] >= 0)
                    t = np.where(cross, d[:, a] / np.where(cross, d[:, a] - d[:, b], 1.0), 0.0)
                    p = c[:, a] + t[:, None] * (c[:, b] - c[:, a])
                    pts.append(p[:, None]); ok.append((cross & ((other[:, a] >= 0) | (other[:, b] >= 0)))[:, None])
            P = np.concatenate(pts, axis=1)
            K = np.concatenate(ok, axis=1)
            side = np.stack([P[..., 0] > P[..., 3], P[..., 0] < -P[..., 3], P[..., 1] > P[..., 3], P[..., 1] < -P[..., 3]], -1)
            keep = ~(np.where(K[..., None], side, True).all(axis=1).any(axis=-1))      # not wholly beyond one side plane
            K &= keep[:, None]
            if not K.any():
                continue
            with np.errstate(divide="ignore", invalid="ignore"):
                nx, ny = P[..., 0] / P[..., 3], P[..., 1] / P[..., 3]
            nx, ny = np.where(K, nx, np.nan), np.where(K, ny, np.nan)
            ext[0] = max(ext[0], np.nanmax(np.abs(nx))); ext[1] = max(ext[1], np.nanmax(np.abs(ny)))
            ext[2] = max(ext[2], np.nanmax(np.nanmax(nx, 1) - np.nanmin(nx, 1))); ext[3] = max(ext[3], np.nanmax(np.nanmax(ny, 1) - np.nanmin(ny, 1)))
    return ext


ENVELOPE_S, ENVELOPE_DS = 2.0 ** 30.5, 2.0 ** 31  # |snapped coordinate| and |difference of two corners|, sub-pixels
MAX_WIDTH = 768                                   # the widest frame mv_create, mv_draw_hires and the debug entries accept


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_product_scenes_stay_inside_the_exact_envelope(scenario):
    """The kernel's integer set-up is exact while every snapped window coordinate has |s| < 2^30.5 sub-pixels and every difference of two
    corners of a triangle is below 2^31 (int32 positions and coefficients, int64 edge constants and bounds; test_raster_conformance_gpu.py
    pins it).  Here the scenarios' own scenes, a few hundred steps of purposeful actions, are measured at 128 x 72 and scaled to the widest
    frame the API accepts, 768 x 4096 (window x = (x_ndc + 1) W / 2; y_ndc scales with the aspect W / H, so both grow with the width
    only).  Vertices made by the near clip lie on w = 0.01, so the measure is the lateral extent of geometry crossing the camera plane:
    the hex mazes set the limit (at 1024 wide their corner differences would pass 2^31)."""
    import helpers

    o = orc.Oracle(scenario, 2, 2)
    o.seed(7)
    o.reset()
    rng = np.random.default_rng(0)
    ext = np.zeros(4)
    for t in range(150):
        o.step(helpers.purposeful_actions(rng, 4, t))
        if t % 3:
            continue
        for e in range(2):
            inst = o.instances(e)
            for a in range(2):
                with np.errstate(all="ignore"), warnings.catch_warnings():
                    warnings.simplefilter("ignore", RuntimeWarning)
                    ext = np.maximum(ext, _window_extent(o.view(e, a), inst))
    o.close()
    Wmax, Hmax = MAX_WIDTH, 4096
    s_max = max((ext[0] + 1) * Wmax / 2 * 256, (ext[1] * (H / W) * Wmax / 2 + Hmax / 2) * 256)
    ds_max = max(ext[2] * Wmax / 2 * 256, ext[3] * (H / W) * Wmax / 2 * 256)
    print("%s: |x_ndc| <= %.1f, |y_ndc| <= %.1f (128 x 72): |s| <= 2^%.2f, |ds| <= 2^%.2f at %d x %d" % (scenario, ext[0], ext[1], np.log2(s_max), np.log2(ds_max), Wmax, Hmax))
    assert s_max < ENVELOPE_S, "window coordinates of %s reach 2^%.2f sub-pixels at %d wide" % (scenario, np.log2(s_max), Wmax)
    assert ds_max < ENVELOPE_DS, "corner differences of %s reach 2^%.2f sub-pixels at %d wide" % (scenario, np.log2(ds_max), Wmax)
