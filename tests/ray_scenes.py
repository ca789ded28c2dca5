"""Constructed scene families for the ray sensors (test infrastructure).  A scene is a dict: views float32[A][16] (world-to-camera,
column-major; agent a casts from views[a]), rows float32[n][18] (mesh, colour, 16 model floats column-major, draw order), tags int32[n]
(a row tagged MV_SEG_AGENT << 8 | a is agent a's own), dirs float32[R][3] (camera space) and max_dist.  Every family is deterministic,
and check_reach(family, scenes, results) asserts from the float64 reference (ray_ref.py) that the scenes reached the case the family is
for, so a scene that drifts away from its case fails instead of passing vacuously."""
import numpy as np

import ray_ref

F32 = np.float32
SEG_STATIC, SEG_OBJECT, SEG_AGENT = 1, 3, 4
EYE = np.eye(4, dtype=F32).reshape(16)


def _row(mesh, m):
    return np.concatenate([[mesh, 0.0], np.asarray(m, dtype=np.float64).T.reshape(-1)]).astype(F32)


def _model(center, half, rot=None):
    m = np.eye(4)
    m[:3, :3] = (np.eye(3) if rot is None else rot) @ np.diag(half)
    m[:3, 3] = center
    return m


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _camera(rng):
    """(view float32[16], camera-to-world float64 4 x 4 rebuilt from the float32 view): a random rigid camera"""
    C = np.eye(4)
    C[:3, :3] = _rot(rng)
    C[:3, 3] = rng.uniform(-20, 20, 3)
    view = np.linalg.inv(C).astype(F32)
    return view.T.reshape(16), np.linalg.inv(view.astype(np.float64))


def grid_dirs(n=16, half=0.35):
    """n x n camera-space directions (not normalised) over a square cone of half-width `half` (tangent) around -z"""
    a = np.linspace(-half, half, n)
    x, y = np.meshgrid(a, a)
    return np.stack([x, y, -np.ones_like(x)], -1).reshape(-1, 3).astype(F32)


def _scene(views, rows, tags, dirs, max_dist=200.0):
    views = np.asarray(views, dtype=F32).reshape(-1, 16)
    rows = np.asarray(rows, dtype=F32).reshape(-1, 18)
    return {"views": views, "rows": rows, "tags": np.asarray(tags, dtype=np.int32).reshape(-1), "dirs": np.asarray(dirs, dtype=F32).reshape(-1, 3),
            "max_dist": float(max_dist)}


def _placed(rng, C, kind, half, rot, span=0.3):
    """a row of mesh `kind` with half extents `half` and rotation `rot` in front of camera C (camera-to-world), inside the grid's cone"""
    D = rng.uniform(3.0, 40.0)
    pc = np.array([rng.uniform(-span, span) * D, rng.uniform(-span, span) * D, -D, 1.0])
    return _row(kind, _model((C @ pc)[:3], half, C[:3, :3] @ rot))


# ---------------------------------------------------------------------------------------------------- families
def boxes(seed=0):
    """boxes axis-aligned to the camera, turned at random, and with per-axis scales from 1e-3 to 1e3"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(24):
        view, C = (EYE, np.eye(4)) if k < 8 else _camera(rng)
        rows = []
        for j in range(6):
            D = rng.uniform(3.0, 40.0)
            if k < 8:
                half, rot = rng.uniform(0.05, 0.3, 3) * D, np.eye(3)
            elif k < 16:
                half, rot = rng.uniform(0.05, 0.3, 3) * D, _rot(rng)
            else:
                half = 10.0 ** rng.uniform(-3, 3, 3)
                half[j % 3] = 10.0 ** rng.uniform(-3, -1)  # a thin axis, the others up to 1e3: plates and needles
                rot = _rot(rng)
            rows.append(_placed(rng, C, 0, half, rot))
        out.append(_scene([view], rows, [SEG_STATIC << 8 | j for j in range(6)], grid_dirs()))
    return out


def meshes(seed=0):
    """capsules, spheres, cones and cylinders under random rigid poses and scales, two to four per scene, some behind others"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(24):
        view, C = _camera(rng)
        kind = 1 + k % 4
        rows = [_placed(rng, C, kind if j == 0 else int(rng.integers(1, 5)), rng.uniform(0.05, 0.25, 3) * 20.0 * rng.uniform(0.2, 1.0), _rot(rng), 0.15)
                for j in range(int(rng.integers(2, 5)))]
        rows.sort(key=lambda r: r[0])
        out.append(_scene([view], rows, [SEG_OBJECT << 8 | j for j in range(len(rows))], grid_dirs()))
    return out


SIGNS = [(-1, 1, 1), (1, -1, 1), (1, 1, -1), (-1, -1, -1), (-1, -1, 1), (1, -1, -1)]


def mirrored(seed=0):
    """every mesh type under one or three negative scales (mirrors) and under two (a rotation), alone ahead of the camera, seen from
    outside and from inside"""
    rng = np.random.default_rng(seed)
    out = []
    for kind in range(5):
        for k, sign in enumerate(SIGNS):
            view, C = _camera(rng)
            D = rng.uniform(4.0, 12.0)
            half = np.array(sign) * rng.uniform(0.4, 0.8, 3) * D * 0.25
            rows = [_row(kind, _model((C @ np.array([0, 0, -D, 1.0]))[:3], half, C[:3, :3] @ _rot(rng)))]
            if k < 2:  # from inside: the camera at the centre of a large one as well
                rows.append(_row(kind, _model(C[:3, 3], np.array(sign) * 50.0, C[:3, :3] @ _rot(rng))))
            out.append(_scene([view], rows, [SEG_OBJECT << 8 | j for j in range(len(rows))], grid_dirs(), 400.0))
    return out


def zero_components(seed=0):
    """axis-aligned boxes (scale 2, integer centres: every object-space value exact) and directions with components of exactly 0, the
    origin inside a slab (o = 0.5), on its border (o = +-1) and outside (o = 1.5), along x and along y"""
    dirs = np.array([[0, 0, -1], [0, 0.25, -1], [0.25, 0, -1], [0, -0.125, -1], [-0.125, 0, -1], [0, 0, 1], [1, 0, 0], [0, 1, 0]], dtype=F32)
    out = []
    for o in (0.5, 1.0, -1.0, 1.5, -1.5, 0.0):
        for axis in (0, 1):
            c = np.zeros(3)
            c[axis] = -2.0 * o  # o_axis = (0 - c) / 2
            c[2] = -10.0
            out.append(_scene([EYE], [_row(0, _model(c, [2.0, 2.0, 2.0]))], [SEG_STATIC << 8], dirs))
    return out


def inside_and_on(seed=0):
    """rays starting inside a box or a mesh, and exactly on a box face (the origin on the planes x = +-1, z = +1 of object space), with
    a wall beyond"""
    rng = np.random.default_rng(seed)
    wall = _row(0, _model([0, 0, -60.0], [200.0, 200.0, 1.0]))
    out = []
    for kind in range(5):
        rows = [_row(kind, _model([0, 0, 0], [3.0, 3.0, 3.0], _rot(rng))), wall]
        out.append(_scene([EYE], rows, [SEG_OBJECT << 8 | 1, SEG_STATIC << 8], grid_dirs(8, 0.8)))
    for c in ([-2.0, 0, 0], [2.0, 0, 0], [0, 0, -2.0], [0, -2.0, 0]):  # scale 2: the origin on a face
        out.append(_scene([EYE], [_row(0, _model(c, [2.0, 2.0, 2.0])), wall], [SEG_OBJECT << 8 | 2, SEG_STATIC << 8], grid_dirs(8, 0.8)))
    return out


def singular(seed=0):
    """rows that are never hit -- a zero scale axis, a NaN and an inf entry -- in front of the same box, before and after it"""
    box = _model([0, 0, -10.0], [4.0, 4.0, 4.0])
    bad = []
    for k in range(3):
        m = box.copy()
        m[k, k] = 0.0
        bad.append(m)
    for v in (np.nan, np.inf, -np.inf):
        m = _model([0, 0, -6.0], [1.0, 1.0, 1.0])
        m[1, 0 if np.isnan(v) else 3] = v
        bad.append(m)
    out = []
    for kind in (0, 2):
        rows = [_row(kind, m) for m in bad] + [_row(0, box)] + [_row(kind, m) for m in bad]
        out.append(_scene([EYE], rows, [SEG_OBJECT << 8 | j for j in range(len(rows))], grid_dirs(8, 0.3)))
    return out


def ties(seed=0, counts=(0, 1, 127, 128, 129, 255, 256, 257, 1200)):
    """exact duplicates (the same row under two tags) at neighbouring entries, across entries 127 | 128 and 255 | 256, within a chunk,
    among filler boxes that no ray hits; instance counts 0, 1, 127, 128, 129, ... and over a thousand"""
    rng = np.random.default_rng(seed)
    dirs = grid_dirs(8, 0.2)
    out = []
    for n in counts:
        rows = [_row(0, _model([rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(5.0, 40.0)], [0.5, 0.5, 0.5])) for _ in range(n)]  # behind
        pairs = [(j, j + 1) for j in (3, 126, 127, 254, 255, 600) if j + 1 < n]
        for p, (a, b) in enumerate(pairs):
            m = _model([rng.uniform(-1, 1), rng.uniform(-1, 1), -5.0 - 3.0 * p], [0.6, 0.6, 0.4], _rot(rng) if p % 2 else None)
            rows[a] = rows[b] = _row(0 if p % 3 else 2, m)
        if n == 1:
            rows = [_row(0, _model([0, 0, -5.0], [1.0, 1.0, 1.0]))]
        out.append(_scene([EYE], rows, [SEG_OBJECT << 8 | (j % 256) for j in range(n)] if n else [], dirs))
    return out


def max_distance(seed=0):
    """a hit at exactly t = 4 and t = 8, cast with max_dist 4, one float32 step below 4, and 8"""
    rows = [_row(0, _model([0, 0, -5.0], [1.0, 1.0, 1.0])), _row(0, _model([3.0, 0, -9.0], [1.0, 1.0, 1.0]))]
    dirs = np.array([[0, 0, -1], [0.125, 0.125, -1], [3.0 / 8.0, 0, -1], [0, 0, -0.5]], dtype=F32)
    return [_scene([EYE], rows, [SEG_STATIC << 8, SEG_STATIC << 8 | 1], dirs, m) for m in (4.0, float(np.nextafter(F32(4.0), F32(0))), 8.0)]


def own_drawables(seed=0):
    """agents 0..7 at one eye, each with a body and eyes of its own in a row ahead: agent a sees through its own to the next one"""
    rows, tags = [], []
    for a in range(8):
        rows.append(_row(1, _model([0, 0, -2.0 - a], [0.3, 0.3, 0.3])))
        rows.append(_row(0, _model([0, 0, -1.8 - a], [0.05, 0.05, 0.05])))
        tags += [SEG_AGENT << 8 | a] * 2
    rows.append(_row(0, _model([0, 0, -40.0], [50.0, 50.0, 1.0])))
    tags.append(SEG_STATIC << 8)
    order = np.argsort([r[0] for r in rows], kind="stable")  # by mesh type, as the engine's lists are
    rows, tags = [rows[i] for i in order], [tags[i] for i in order]
    return [_scene([EYE] * 8, rows, tags, grid_dirs(4, 0.01))]


FAMILIES = {"boxes": boxes, "meshes": meshes, "mirrored": mirrored, "zero_components": zero_components, "inside_and_on": inside_and_on,
            "singular": singular, "ties": ties, "max_distance": max_distance, "own_drawables": own_drawables}


# ---------------------------------------------------------------------------------------------------- rays at shared edges
def front_edge_targets(kind, C, model, facing=0.2):
    """the world points, midpoints of edges and shared vertices, where front-facing triangles of mesh `kind` meet, seen from the camera
    at C (camera-to-world), with the facing margin (|cos| of normal and ray) at least `facing` for every triangle that meets there.  The
    tables repeat a position under several normals, so corners are matched by position, not by index."""
    P, I = ray_ref.mesh(kind)
    _, key = np.unique(P, axis=0, return_inverse=True)
    key = key.reshape(-1)
    M = np.asarray(model, dtype=np.float64)
    W = P @ M[:3, :3].T + M[:3, 3]
    n = np.cross(W[I[:, 1]] - W[I[:, 0]], W[I[:, 2]] - W[I[:, 0]])
    nn = np.linalg.norm(n, axis=1)
    tris = np.nonzero(nn > 0)[0]  # the tables' zero-area triangles touch nothing
    d = W[I].mean(axis=1) - C[:3, 3]
    cos = np.zeros(len(I))
    cos[tris] = -(n[tris] * d[tris]).sum(1) / (nn[tris] * np.linalg.norm(d[tris], axis=1))
    good = cos >= facing
    edges, around, pos = {}, {}, {}
    for t in tris:
        for a, b in ((0, 1), (1, 2), (2, 0)):
            e = tuple(sorted((int(key[I[t, a]]), int(key[I[t, b]]))))
            edges.setdefault(e, []).append(t)
            pos[e] = (W[I[t, a]] + W[I[t, b]]) / 2
        for a in range(3):
            around.setdefault(int(key[I[t, a]]), []).append(t)
            pos[int(key[I[t, a]])] = W[I[t, a]]
    pts = [pos[e] for e, ts in edges.items() if len(ts) == 2 and all(good[t] for t in ts)]
    pts += [pos[v] for v, ts in around.items() if len(ts) >= 3 and all(good[t] for t in ts)]
    return np.array(pts).reshape(-1, 3)


def edge_scenes(poses=20, seed=0, far=False):
    """per mesh type, `poses` random poses: one instance ahead of a random camera and rays aimed (camera space) at the midpoints of the
    edges and at the vertices where front faces meet; far: small meshes 30 to 100 units away"""
    rng = np.random.default_rng(seed)
    out = []
    for kind in range(1, 5):
        for p in range(poses):
            view, C = _camera(rng)
            D = rng.uniform(30.0, 100.0) if far else rng.uniform(3.0, 20.0)
            # far: small meshes (scale 0.01 .. 0.45), so that the origin is hundreds to thousands of object units away
            half = rng.uniform(0.3, 1.5, 3) * (rng.choice([0.03, 0.3]) if far else D * 0.1)
            m = _model((C @ np.array([0, 0, -D, 1.0]))[:3], half, C[:3, :3] @ _rot(rng))
            row = _row(kind, m)
            M32 = row[2:].astype(np.float64).reshape(4, 4).T
            pts = front_edge_targets(kind, C, M32)
            Cinv = np.linalg.inv(C)
            dirs = pts @ Cinv[:3, :3].T + Cinv[:3, 3]
            for k in range(0, len(dirs), 256):
                out.append(_scene([view], [row], [SEG_OBJECT << 8 | kind], dirs[k:k + 256], 400.0))
    return out


def check_reach(family, scenes, results):
    """results[s][a]: ray_ref.Result of scene s, agent a"""
    hits = sum(int((r.tag != 0).sum()) for rs in results for r in rs)
    rays = sum(r.tag.size for rs in results for r in rs)
    if family in ("boxes", "meshes"):
        assert hits >= rays // 8, "%s: %d of %d rays hit" % (family, hits, rays)
        if family == "boxes":
            conds = [r.cond[r.tag != 0].max(initial=1.0) for rs in results for r in rs]
            assert max(conds) > 1e4, "an anisotropic box is hit"
    elif family == "mirrored":
        for s, rs in zip(scenes, results):
            assert (rs[0].tag != 0).any(), "every mirrored instance is hit"
        assert sum(1 for s in scenes if np.linalg.det(s["rows"][0, 2:].reshape(4, 4)[:3, :3].astype(np.float64)) < 0) >= 15
    elif family == "zero_components":
        assert any((r.tag != 0).any() for rs in results for r in rs) and any((r.tag == 0).any() for rs in results for r in rs)
    elif family == "inside_and_on":
        for s, rs in zip(scenes, results):
            assert (rs[0].tag == SEG_STATIC << 8).all(), "from inside, or from a face, the wall is seen through the instance"
    elif family == "singular":
        for rs in results:
            assert (rs[0].tag == SEG_OBJECT << 8 | 6).all(), "only the finite box is hit"
    elif family == "ties":
        for s, rs in zip(scenes, results):
            if len(s["rows"]) > 1:
                assert (rs[0].gap[rs[0].tag != 0] == 0).sum() > 0, "exact ties"
    elif family == "max_distance":
        assert results[0][0].tag[0] != 0 and results[1][0].tag[0] == 0 and results[0][0].dist[0] == 4.0
    elif family == "own_drawables":
        for a, r in enumerate(results[0]):
            assert (r.tag == (SEG_AGENT << 8 | (1 if a == 0 else 0))).all(), "agent %d sees the nearest drawable not its own" % a
