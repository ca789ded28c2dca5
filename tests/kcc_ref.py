"""Float64 reference of the character controller's collision queries (DESIGN.md section 6), independent of the product's arithmetic.

The product and the oracle solve each of a box's 23 boundary features in closed form in float32.  Here the same contact is found
from the float64 signed distance alone, with no feature enumeration:

* sweep: the capsule axis midpoint moves from `from` to `to`; a collider is met where the signed distance to its inflated shape
  (box: the box grown by the capsule's segment, rounded by r - 0.04; agent: the capsule of half length 2 hh and radius 2 r - 0.04) first
  reaches 0.  The root is bracketed by dense sampling of the path and bisected; the normal is the distance's gradient there, and the
  feature is read off the region of the box the closest point lies in.  A start already inside is a hit at t = 0 when the path runs into
  the surface (dot(d, n0) < -FLT_EPSILON), as the callback defines it.
* recover: the first collider in collider order whose unrounded signed distance is below -0.041 pushes the point out along its gradient.

Each answer carries margins: how far the case is from a decision the float32 code could take the other way (a graze, a start on the
surface, a feature boundary, a tie between colliders, the slope filter, the penetration threshold).  Agreement is asserted only where
every margin clears the bound the tests state."""
import numpy as np

R = 0.33
HH = 1.05 / 2
RHO_BOX = R - 0.04
RHO_CAP = 2 * R - 0.04
EPS = float(np.float32(1.1920929e-07))
MAX_PEN = float(np.float32(0.041))
SAMPLES = 4096


def _to_local(col, p):
    if col["axes"] is None:
        return np.array(p, dtype=np.float64)
    ax, az = col["axes"]
    return np.array([p[0] * ax + p[2] * az, p[1], -p[0] * az + p[2] * ax])


def _to_world(col, n):
    if col["axes"] is None:
        return np.array(n, dtype=np.float64)
    ax, az = col["axes"]
    return np.array([n[0] * ax - n[2] * az, n[1], n[0] * az + n[2] * ax])


def _box_sd(o, H):
    """signed distance of local point o to the box of half extents H, its gradient, and the closest point's region margin"""
    q = np.abs(o) - H
    if np.all(q <= 0):
        ax = int(np.argmax(q))
        n = np.zeros(3)
        n[ax] = 1.0 if o[ax] >= 0 else -1.0
        srt = np.sort(q)
        return float(q[ax]), n, float(srt[2] - srt[1])  # margin: the gap to the axis tie
    e = np.maximum(q, 0.0)
    d = float(np.linalg.norm(e))
    n = np.sign(o) * e / d
    return d, n, float(np.min(np.abs(q)))  # margin: how far the closest point is from the next region


def _cap_sd(o, L):
    cy = min(max(o[1], -L), L)
    e = np.array([o[0], o[1] - cy, o[2]])
    d = float(np.linalg.norm(e))
    return d, (e / d if d > 0 else np.array([1.0, 0.0, 0.0])), d


def distance(col, p, rounded=True):
    """(signed distance, world gradient, region margin) of the capsule centre p against one collider: rounded = the sweep's inflated
    shape, else recovery's (box grown by the segment minus r; capsule distance minus 2 r)"""
    c = np.array(col["c"], dtype=np.float64)
    if col["kind"] == "box":
        H = np.array(col["h"], dtype=np.float64) + np.array([0.0, HH, 0.0])
        d, n, m = _box_sd(_to_local(col, p - c), H)
        return d - (RHO_BOX if rounded else R), _to_world(col, n), m
    d, n, m = _cap_sd(p - c, 2 * HH)
    return d - (RHO_CAP if rounded else 2 * R), n, m


def _sd_many(col, pts):
    """the rounded signed distance of many points at once (sampling only; the root itself is refined with distance())"""
    o = pts - np.array(col["c"], dtype=np.float64)[None, :]
    if col["kind"] == "box":
        if col["axes"] is not None:
            ax, az = col["axes"]
            o = np.stack([o[:, 0] * ax + o[:, 2] * az, o[:, 1], -o[:, 0] * az + o[:, 2] * ax], axis=1)
        q = np.abs(o) - (np.array(col["h"], dtype=np.float64) + np.array([0.0, HH, 0.0]))[None, :]
        inside = np.all(q <= 0, axis=1)
        return np.where(inside, q.max(axis=1), np.linalg.norm(np.maximum(q, 0.0), axis=1)) - RHO_BOX
    cy = np.clip(o[:, 1], -2 * HH, 2 * HH)
    return np.sqrt(o[:, 0] ** 2 + (o[:, 1] - cy) ** 2 + o[:, 2] ** 2) - RHO_CAP


def feature_of(col, p):
    """the device's feature number of the box region the closest point to p lies in (0 for capsules)"""
    if col["kind"] != "box":
        return 0
    H = np.array(col["h"], dtype=np.float64) + np.array([0.0, HH, 0.0])
    o = _to_local(col, p - np.array(col["c"], dtype=np.float64))
    out = np.abs(o) > H
    k = int(out.sum())
    if k <= 1:
        return int(np.argmax(out)) if k == 1 else 0
    if k == 2:
        kk = int(np.argmin(out))
        i, j = (kk + 1) % 3, (kk + 2) % 3
        return 3 + 4 * kk + (2 if o[i] > 0 else 0) + (1 if o[j] > 0 else 0)
    return 15 + (4 if o[0] > 0 else 0) + (2 if o[1] > 0 else 0) + (1 if o[2] > 0 else 0)


def first_contact(col, a, b):
    """first t in [0, 1] at which the path a -> b meets the collider's inflated shape: (t or None, normal, feature, margins dict)"""
    d = b - a
    L = float(np.linalg.norm(d))
    s0, n0, m0 = distance(col, a)
    if s0 <= 0:
        dn = float(np.dot(d, n0))
        marg = {"start": -s0, "inside": abs(dn + EPS), "region": m0 if col["kind"] == "box" else np.inf}
        return (0.0 if dn < -EPS else None), n0, 0, marg
    ts = np.linspace(0.0, 1.0, SAMPLES + 1)
    sd = _sd_many(col, a[None, :] + ts[:, None] * d[None, :])
    i = int(np.argmax(sd <= 0)) if np.any(sd <= 0) else -1
    # grazing margin: the least distance along the path when it misses, the deepest reach past the surface when it hits (refined
    # around the best sample by golden-section search)
    j = int(np.argmin(sd))
    lo, hi = ts[max(j - 1, 0)], ts[min(j + 1, SAMPLES)]
    g = (np.sqrt(5) - 1) / 2
    for _ in range(60):
        x1, x2 = hi - g * (hi - lo), lo + g * (hi - lo)
        if distance(col, a + x1 * d)[0] < distance(col, a + x2 * d)[0]:
            hi = x2
        else:
            lo = x1
    smin = min(float(sd[j]), distance(col, a + 0.5 * (lo + hi) * d)[0])
    marg = {"start": s0, "graze": abs(smin)}
    if i < 0:
        return None, None, -1, marg
    lo, hi = ts[i - 1], ts[i]
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if distance(col, a + mid * d)[0] <= 0:
            hi = mid
        else:
            lo = mid
    t = hi
    p = a + t * d
    _, n, m = distance(col, p)
    marg["region"] = m if col["kind"] == "box" else np.inf
    marg["end"] = (1.0 - t) * L  # the callback keeps only fractions below the current best, 1 to start with
    return t, n, feature_of(col, p), marg


def sweep(case):
    """the reference answer of a sweep case: dict hit, index, t, normal, feature, L (= |d|) and the least margin (length units)"""
    q = case.query
    a, b = np.array(q[0:3], dtype=np.float64), np.array(q[3:6], dtype=np.float64)
    fdir, mind = np.array(q[6:9], dtype=np.float64), float(q[9])
    L = float(np.linalg.norm(b - a))
    cols = case.colliders()
    self_idx = len(cols) - case.A + case.agent
    hits, margins = [], []
    for idx, col in enumerate(cols):
        if idx == self_idx or not col["enabled"]:
            continue
        t, n, f, m = first_contact(col, a, b)
        margins.append(min(m.values()))
        if t is None:
            continue
        slope = float(np.dot(fdir, n)) - mind
        margins.append(abs(slope))
        if slope >= 0:
            hits.append((t, idx, n, f))
    res = {"hit": False, "index": -1, "t": 1.0, "normal": np.zeros(3), "feature": -1, "L": L}
    if hits:
        hits.sort(key=lambda h: (h[0], h[1]))
        t, idx, n, f = hits[0]
        res.update(hit=True, index=idx, t=t, normal=n, feature=f)
        if len(hits) > 1:
            margins.append((hits[1][0] - t) * L)
    res["margin"] = min(margins) if margins else np.inf
    return res


def recover(case):
    """the reference answer of a recovery case: dict pen, index, delta and the least margin"""
    p = np.array(case.query[0:3], dtype=np.float64)
    cols = case.colliders()
    self_idx = len(cols) - case.A + case.agent
    margins = []
    for idx, col in enumerate(cols):
        if idx == self_idx or not col["enabled"]:
            continue
        s, n, m = distance(col, p, rounded=False)
        margins.append(abs(s + MAX_PEN))
        if s < -MAX_PEN:
            if s + R <= 0 or col["kind"] != "box":
                margins.append(m)  # inside the box proper (or a capsule): the normal's own decision
            return {"pen": True, "index": idx, "delta": n * -s, "margin": min(margins)}
    return {"pen": False, "index": -1, "delta": np.zeros(3), "margin": min(margins) if margins else np.inf}
