"""An independent restatement of the ray sensors' hit rules (DESIGN.md section 3, "Ray sensors") in float64, for tests.

Same rules as the kernel and tests/oracle_seg/orc_rays.cpp, different arithmetic: the float32 inputs are widened to float64 and inverted
with np.linalg.inv; boxes are intersected face by face (the plane of each face, then whether the point lies on the face); other meshes by
a plane hit and a 2 x 2 barycentric solve, facing judged by the sign of n . v times the model's handedness.  The same inclusive tie rule
(a later row wins an exact tie), the own-drawable skip, the inclusive max distance and the widened barycentric bounds (EDGE_TOL, taken
only when no triangle of the instance is hit within the exact bounds) apply.
The mesh tables come from the oracle (data, not arithmetic).

Besides the hit, every ray gets margins that say how far it is from a decision: the gap from the winner to the nearest candidate of
another row, the distance of a deciding hit point to the edge of its face (object units; negative outside the face), the facing margin
(|cos| between the face normal and the ray), the distance of a candidate to the ray's origin, and |t - max_dist|."""
import numpy as np

import orc

EDGE_TOL = 2.0 ** -18  # the widening of the barycentric bounds per object unit of |o - p0|_1, plus one (DESIGN.md section 3, step 4)
_MESHES = {}


def mesh(kind):
    """(vertex positions float64 [n][3], triangle indices [t][3]) of mesh type kind 1..4, from the oracle's tables"""
    if kind not in _MESHES:
        vtx, idx = orc.mesh(kind)
        _MESHES[kind] = (vtx.view(np.float32).reshape(-1, 6)[:, :3].astype(np.float64), idx.reshape(-1, 3).astype(np.int64))
    return _MESHES[kind]


def _mat(m16):
    """a column-major float32[16] as a float64 4 x 4 matrix [row][col]"""
    return np.asarray(m16, dtype=np.float32).astype(np.float64).reshape(4, 4).T


def model_info(inst18):
    """(inverse float64 4x4 or None for a singular / non-finite model, mirrored, 2-norm condition number of the 3 x 3 part)"""
    M = _mat(np.asarray(inst18, dtype=np.float32)[2:18])
    if not np.isfinite(M).all():
        return None, False, np.inf
    A = M[:3, :3]
    det = np.linalg.det(A)
    if det == 0.0:
        return None, False, np.inf
    cond = np.linalg.cond(A)
    if not np.isfinite(cond) or cond > 1e12:
        return None, False, np.inf
    return np.linalg.inv(M), bool(det < 0.0), float(cond)


class Result:
    """dist float64[R] (0 = no hit), tag int64[R], row int64[R] (-1 = none), cond float64[R] (the winner's condition number, 1 for no
    hit) and margins gap, edge, facing, origin, maxd float64[R] (inf where nothing bears on the decision)"""

    def __init__(self, R):
        self.dist = np.zeros(R)
        self.tag = np.zeros(R, dtype=np.int64)
        self.row = np.full(R, -1, dtype=np.int64)
        self.cond = np.ones(R)
        for k in ("gap", "edge", "facing", "origin", "maxd"):
            setattr(self, k, np.full(R, np.inf))

    def robust(self, gap=1e-4, edge=1e-3, facing=1e-3, origin=1e-4, maxd=1e-5):
        """rays every margin of which clears the thresholds (gap, origin and maxd relative to t, edge in object units)"""
        t = np.maximum(self.dist, 1e-30)
        return (self.gap > gap * t) & (self.edge > edge) & (self.facing > facing) & (self.origin > origin) & (self.maxd > maxd * t)


def _box_candidates(o, v, mirrored):
    """per ray: (t or nan, edge margin, origin margin) of a box [-1, 1]^3 in object space, face by face.  A face is the plane x_i = +-1;
    the ray meets it at t = (+-1 - o_i) / v_i, and the face counts when the point lies within [-1, 1] on the other two axes and the ray
    enters there (v_i pointing inwards) -- or, mirrored, leaves there.  The edge margin is the point's distance to the face's border."""
    R = o.shape[0]
    best_t = np.full(R, np.nan)
    best_e = np.full(R, -np.inf)
    near_e = np.full(R, np.inf)  # |distance to the border| of every face crossing near the ray (a near miss decides as much as a hit)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(3):
            others = [j for j in range(3) if j != i]
            for side in (-1.0, 1.0):
                t = (side - o[:, i]) / v[:, i]
                p = o + t[:, None] * v
                e = np.min(1.0 - np.abs(p[:, others]), axis=1)
                entering = v[:, i] * side < 0.0  # moving towards the inside across this face
                counts = (~entering) if mirrored else entering
                ok = counts & np.isfinite(t) & (v[:, i] != 0.0)
                near_e = np.where(ok & (t > 0.0) & np.isfinite(e), np.minimum(near_e, np.abs(e)), near_e)
                hit = ok & (e >= 0.0)
                take = hit & (np.isnan(best_t) | (e > best_e))
                best_t = np.where(take, t, best_t)
                best_e = np.where(take, e, best_e)
    # an axis the ray runs parallel to: inside its slab or not decides alone
    for i in range(3):
        par = v[:, i] == 0.0
        near_e = np.where(par, np.minimum(near_e, np.abs(1.0 - np.abs(o[:, i]))), near_e)
        best_t = np.where(par & (np.abs(o[:, i]) > 1.0), np.nan, best_t)
    origin = np.where(np.isnan(best_t), np.inf, np.abs(best_t))
    return best_t, near_e, origin


def _mesh_candidates(o, v, kind, mirrored):
    """per ray: (nearest t or nan, edge margin, facing margin, origin margin) over the front faces of mesh `kind`"""
    P, I = mesh(kind)
    p0, p1, p2 = P[I[:, 0]], P[I[:, 1]], P[I[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    n = np.cross(e1, e2)  # counter-clockwise normal
    nn = np.linalg.norm(n, axis=1)
    keep = nn > 0.0  # a triangle of zero area (the tables' poles) faces nothing: det = 0 in the kernel
    p0, p1, p2, e1, e2, n, nn = p0[keep], p1[keep], p2[keep], e1[keep], e2[keep], n[keep], nn[keep]
    G = np.stack([np.stack([(e1 * e1).sum(1), (e1 * e2).sum(1)], -1), np.stack([(e1 * e2).sum(1), (e2 * e2).sum(1)], -1)], -2)  # [T][2][2]
    Ginv = np.linalg.inv(G)
    s = -1.0 if mirrored else 1.0
    vn = v @ n.T  # [R][T]
    front = s * vn < 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        t = ((p0 * n).sum(1)[None, :] - o @ n.T) / vn  # plane hit: n . (o + t v - p0) = 0
        q = o[:, None, :] + t[:, :, None] * v[:, None, :] - p0[None]  # [R][T][3]
        rhs = np.stack([(q * e1[None]).sum(-1), (q * e2[None]).sum(-1)], -1)
        ab = np.einsum("tij,rtj->rti", Ginv, rhs)
    a, b = ab[..., 0], ab[..., 1]
    tol = EDGE_TOL * (1.0 + np.abs(o[:, None, :] - p0[None]).sum(-1))  # [R][T]
    exact = (a >= 0.0) & (a <= 1.0) & (b >= 0.0) & (a + b <= 1.0)
    inside = (a >= -tol) & (a <= 1.0 + tol) & (b >= -tol) & (a + b <= 1.0 + tol)
    # signed distance of the plane hit to the three edge lines (object units): barycentric times the opposite edge's height
    h0 = nn / np.linalg.norm(p2 - p1, axis=1)  # height over edge p1p2 (barycentric 1 - a - b)
    h1 = nn / np.linalg.norm(e2, axis=1)       # over p0p2 (a)
    h2 = nn / np.linalg.norm(e1, axis=1)       # over p0p1 (b)
    edge = np.minimum(np.minimum(a * h1[None], b * h2[None]), (1.0 - a - b) * h0[None])
    cosv = np.abs(vn) / (nn[None] * np.linalg.norm(v, axis=1)[:, None])
    cand = front & inside & (t > 0.0) & np.isfinite(t)
    hit_exact = (cand & exact).any(axis=1)
    cand = np.where(hit_exact[:, None], cand & exact, cand)  # the widened bounds only where no triangle is hit within the exact ones
    tt = np.where(cand, t, np.inf)
    k = np.argmin(tt, axis=1)
    r = np.arange(o.shape[0])
    best = tt[r, k]
    best = np.where(np.isfinite(best), best, np.nan)
    # margins over the faces whose plane hit lies near the triangle and not behind the best hit: those decide
    lim = np.where(np.isnan(best), np.inf, best)[:, None] * (1.0 + 1e-6)
    near = np.isfinite(t) & (t <= lim) & (edge > -1e-2)
    e_m = np.where(near & front & (t > 0.0), np.abs(edge), np.inf).min(axis=1)
    f_m = np.where(near & (t > 0.0) & (edge > -1e-3), cosv, np.inf).min(axis=1)
    o_m = np.where(near & front & (edge > -1e-3), np.abs(t), np.inf).min(axis=1)
    return best, e_m, f_m, o_m


def cast(view16, inst18, tags, dirs, max_dist, agent=-1):
    """rays `dirs` (camera space) of one caster seen through view16 against rows inst18 with their tags, in float64: a Result"""
    inst18 = np.asarray(inst18, dtype=np.float32).reshape(-1, 18)
    tags = np.asarray(tags, dtype=np.int64).reshape(-1)
    d = np.asarray(dirs, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    R = d.shape[0]
    cam = np.linalg.inv(_mat(view16))
    ow = cam[:3, 3]
    dw = d @ cam[:3, :3].T
    own = -1 if agent < 0 else (4 << 8 | agent)
    maxd = float(np.float32(max_dist))
    cands = []  # (row, t[R] with nan for none, edge, facing, origin)
    for i in range(inst18.shape[0]):
        if tags[i] == own:
            continue
        inv, mirrored, cond = model_info(inst18[i])
        if inv is None:
            continue
        o = np.broadcast_to(inv[:3, :3] @ ow + inv[:3, 3], (R, 3))
        v = dw @ inv[:3, :3].T
        kind = int(inst18[i, 0])
        if kind == 0:
            t, e, org = _box_candidates(o, v, mirrored)
            f = np.full(R, np.inf)
        else:
            t, e, f, org = _mesh_candidates(o, v, kind, mirrored)
        cands.append((i, t, e, f, org, cond))
    res = Result(R)
    best = np.full(R, maxd)
    for i, t, e, f, org, cond in cands:  # draw order; a later row wins an exact tie
        take = np.isfinite(t) & (t > 0.0) & (t <= best)
        best = np.where(take, t, best)
        res.row = np.where(take, i, res.row)
        res.cond = np.where(take, cond, res.cond)
    hit = res.row >= 0
    res.dist = np.where(hit, best, 0.0)
    res.tag = np.where(hit, tags[np.maximum(res.row, 0)], 0) if len(tags) else res.tag
    lim = np.where(hit, best, maxd) * (1.0 + 1e-6)
    for i, t, e, f, org, cond in cands:
        relevant = np.where(np.isnan(t), True, t <= lim)  # a near miss or a hit not behind the winner
        res.edge = np.where(relevant, np.minimum(res.edge, e), res.edge)
        res.facing = np.where(relevant, np.minimum(res.facing, f), res.facing)
        res.origin = np.where(relevant, np.minimum(res.origin, org), res.origin)
        other = np.isfinite(t) & (res.row != i)
        res.gap = np.where(other & hit, np.minimum(res.gap, np.abs(t - best)), res.gap)
        res.maxd = np.where(np.isfinite(t), np.minimum(res.maxd, np.abs(t - maxd)), res.maxd)
    return res
