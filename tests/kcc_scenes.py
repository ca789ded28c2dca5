"""Constructed contact cases for the character controller's collision code (mv_debug_kcc, the oracle's orc_kcc_case, kcc_ref).

A Case is one collider set in collider order (statics before the objects, the objects, the other statics, the agents' capsules) and
one query by one agent.  Each family builds its cases and asserts, from the float64 reference (kcc_ref), that it reaches what it is
named for; the tests then run every family through the device, the oracle and the reference."""
import math

import numpy as np

import kcc_ref

F32 = np.float32
MAX_OBJ, MAX_AG = 128, 8
SWEEP, RECOVER, STEP = 0, 1, 2
DT = float(F32(1.0) / F32(15.0))
MAX_SLOPE_COS = float(F32(math.cos(F32(45.0) * F32(math.pi / 180.0))))
RHO = kcc_ref.RHO_BOX
HH = kcc_ref.HH


def f32(v):
    return float(F32(v))


def yaw_axes(deg):
    """a rotated static's local x axis (ax, az) as float32 cos / sin of the angle, as the hex mazes compute it"""
    a = F32(deg) * F32(math.pi / 180.0)
    return float(F32(math.cos(a))), float(F32(math.sin(a)))


class Case:
    def __init__(self, mode, A=1, agent=0, pos=(0.0, 0.0, 0.0)):
        self.mode, self.A, self.agent = mode, A, agent
        self.statics, self.objects = [], []  # (c, h, solid / enabled, axes or None)
        self.n_static_pre = 0
        self.agents = [[0.0, 50.0 + 5 * i, 0.0] for i in range(A)]  # out of the way unless placed
        self.agents[agent] = [f32(v) for v in pos]
        self.query = [0.0] * 20

    def box(self, c, h, solid=True, axes=None):
        """a static box; returns its collider index once the case is complete (n_static_pre = 0: after the objects)"""
        self.statics.append(([f32(v) for v in c], [f32(v) for v in h], solid, axes))
        return len(self.statics) - 1

    def obj(self, c, h, enabled=True):
        self.objects.append(([f32(v) for v in c], [f32(v) for v in h], enabled, None))

    def static_index(self, j):
        return j if j < self.n_static_pre else j + len(self.objects)

    def sweep(self, a, b, fdir=(0.0, 0.0, 0.0), min_dot=-1.0):
        self.query[0:10] = [f32(v) for v in list(a) + list(b) + list(fdir)] + [f32(min_dot)]
        return self

    def recover(self, p):
        self.query[0:3] = [f32(v) for v in p]
        return self

    def step(self, pos, hvel=(0, 0, 0), vvel=0.0, voff=0.0, step_off=0.0, jump_speed=10.0, was_on_ground=False, was_jumping=False):
        self.agents[self.agent] = [f32(v) for v in pos]
        self.query[0:17] = [f32(v) for v in list(pos) + list(hvel) + [vvel, voff, step_off, jump_speed, 0.0, 1.0, 0.0]] + [
            float(was_on_ground), float(was_jumping), DT, MAX_SLOPE_COS]
        return self

    def colliders(self):
        out = []
        def add(rows):
            for c, h, on, axes in rows:
                out.append({"kind": "box", "c": c, "h": h, "enabled": on, "axes": axes})
        add(self.statics[: self.n_static_pre])
        add(self.objects)
        add(self.statics[self.n_static_pre:])
        for p in self.agents:
            out.append({"kind": "cap", "c": list(p), "h": [0, 0, 0], "enabled": True, "axes": None})
        return out


def pack(cases):
    n = len(cases)
    hdr = np.zeros((n, 8), np.int32)
    boxes = np.zeros((n, 2 * MAX_OBJ, 10), np.float32)
    agents = np.zeros((n, MAX_AG, 3), np.float32)
    query = np.zeros((n, 20), np.float32)
    for k, cs in enumerate(cases):
        hdr[k, :6] = [cs.n_static_pre, len(cs.statics), len(cs.objects), cs.A, cs.mode, cs.agent]
        for j, (c, h, on, axes) in enumerate(cs.statics):
            boxes[k, j] = c + h + [float(on), float(axes is not None)] + list(axes or (1.0, 0.0))
        for j, (c, h, on, _) in enumerate(cs.objects):
            boxes[k, MAX_OBJ + j] = c + h + [float(on), 0.0, 1.0, 0.0]
        agents[k, : cs.A] = cs.agents
        query[k] = cs.query
    return hdr, boxes, agents, query


def _to_world(axes, v):
    if axes is None:
        return np.array(v, dtype=np.float64)
    ax, az = axes
    return np.array([v[0] * ax - v[2] * az, v[1], v[0] * az + v[2] * ax])


def feature_normal(f, rng):
    """a local outward normal in the interior of feature f's region, and the box-surface point's sign pattern (which axes sit at +-H)"""
    n = np.zeros(3)
    sel = np.zeros(3)
    if f < 3:
        n[f] = rng.choice([-1.0, 1.0])
        sel[f] = n[f]
    elif f < 15:
        e = f - 3
        k = e >> 2
        i, j = (k + 1) % 3, (k + 2) % 3
        si, sj = (1.0 if e & 2 else -1.0), (1.0 if e & 1 else -1.0)
        th = rng.uniform(0.2, 1.37)
        n[i], n[j] = si * math.cos(th), sj * math.sin(th)
        sel[i], sel[j] = si, sj
    else:
        e = f - 15
        s = np.array([(1.0 if e & 4 else -1.0), (1.0 if e & 2 else -1.0), (1.0 if e & 1 else -1.0)])
        v = rng.uniform(0.3, 1.0, 3)
        n = s * v / np.linalg.norm(v)
        sel = s
    return n, sel


def place_feature(cs, f, H, axes, target, d, rng):
    """add a static box whose inflated shape the path through `target` along d first meets at feature f, at `target`; H is the
    box's half extents (without the capsule segment).  d must oppose the chosen normal, which is drawn until it does."""
    Hs = np.array(H, dtype=np.float64) + np.array([0.0, HH, 0.0])
    for _ in range(200):
        n, sel = feature_normal(f, rng)
        if f < 3:
            # the face pair whose normal opposes the motion
            loc_d = kcc_ref._to_local({"axes": axes}, d) if axes is not None else d
            if loc_d[f] == 0:
                return None
            n[f] = -math.copysign(1.0, loc_d[f])
            sel[f] = n[f]
        nw = _to_world(axes, n)
        if np.dot(nw, d) < -0.2 * np.linalg.norm(d):
            break
    else:
        return None
    surf = np.where(sel != 0, sel * Hs, rng.uniform(-0.6, 0.6, 3) * Hs)  # a point of that feature, away from its ends
    local = surf + RHO * n
    c = np.asarray(target, dtype=np.float64) - _to_world(axes, local)
    return cs.box(c, H, True, axes)


YAWS = [0.0, 90.0, -90.0, 180.0, 30.0, 45.0, 60.0, 120.0, 240.0, 300.0]


def family_features(seed=1):
    """each of the 23 box features as the first contact, half extents 0.05 to 50, yaws 0, +-90, 180, 30, 45 and the hex mazes' 60s"""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(23):
        for yaw in YAWS:
            for _ in range(2):
                while True:  # a direction that can meet feature f first
                    H = np.exp(rng.uniform(math.log(0.05), math.log(50.0), 3))
                    d = rng.normal(size=3)
                    d *= rng.uniform(0.3, 2.5) / np.linalg.norm(d)
                    cs = Case(SWEEP)
                    axes = None if yaw == 0.0 and rng.random() < 0.5 else yaw_axes(yaw)
                    t = rng.uniform(0.1, 0.9)
                    if place_feature(cs, f, H, axes, t * d, d, rng) is not None:
                        break
                cs.sweep((0, 0, 0), d)
                cs.want = {"index": 0, "feature": f, "yaw": yaw}
                out.append(cs)
    return out


def family_decode(seed=2, counts=range(1, 33)):
    """n live candidates, each met at its own feature and fraction, the winner each of them in turn: every live count through the
    (candidate x feature) decode"""
    rng = np.random.default_rng(seed)
    d = np.array([1.3, -0.55, 0.8])
    reach = [f for f in range(23)]
    out = []
    for n in counts:
        for w in range(n):
            cs = Case(SWEEP)
            ts = np.linspace(0.25, 0.95, n)
            rng.shuffle(ts)
            ts[[w, int(np.argmin(ts))]] = ts[[int(np.argmin(ts)), w]]
            ts[w] = 0.15
            ok = True
            for j in range(n):
                H = rng.uniform(0.05, 0.3, 3)
                for k in range(23):
                    f = reach[(j + k + n) % 23]
                    if place_feature(cs, f, H, None, ts[j] * d, d, rng) is not None:
                        break
                else:
                    ok = False
            if not ok:
                continue
            cs.sweep((0, 0, 0), d)
            cs.want = {"index": w}
            out.append(cs)
    return out


def family_counts():
    """0 .. 97+ candidates, all live, the nearest at the first and at the last slot: the chunk loop and the MV_MAX_CAND cap"""
    out = []
    d = np.array([2.0, 0.0, 0.0])
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 96, 97, 100, 128):
        for nearest in ("first", "last"):
            cs = Case(SWEEP)
            for j in range(n):
                rank = j if nearest == "first" else n - 1 - j
                x = 0.4 + 1.4 * rank / max(n, 1)
                cs.box((x + RHO + 0.01, 0.15 * ((j % 5) - 2), 0.005 * ((j % 7) - 3)), (0.01, 0.02, 0.02))
            cs.sweep((0, 0, 0), d)
            cs.want = {"index": (0 if nearest == "first" else n - 1) if n else -1, "count": n}
            out.append(cs)
    return out


def family_ties():
    """two or three colliders met at the same fraction, at candidate slots 0|1, 31|32, 63|64 and 94|95: duplicate boxes, rotated boxes,
    a floor seam, capsules; and t = 0 ties whose lower index the slope filter rejects"""
    out = []
    for slot in (0, 31, 63, 94):
        for kind in ("dup", "rot", "seam", "cap", "filtered"):
            A = 3 if kind == "cap" else 1
            cs = Case(SWEEP, A=A, agent=0)
            for j in range(slot):  # fillers before the tied pair: in the envelope, outside the sweep's bounds
                filler(cs, j)
            if kind == "dup":
                first = [cs.box((1.0 + RHO + 0.1, 0.0, 0.0), (0.1, 0.5, 0.5)) for _ in range(2 if slot == 94 else 3)][0]
                cs.sweep((0, 0, 0), (1.5, 0.0, 0.05))
            elif kind == "rot":
                ax = yaw_axes(60.0)
                first = [cs.box((1.2, 0.0, 0.1), (0.1, 0.5, 0.5), axes=ax) for _ in range(2)][0]
                cs.sweep((0, 0, 0), (1.5, 0.0, 0.05))
            elif kind == "seam":
                first = cs.box((-0.5, -1.0, 0.0), (0.5, 0.25, 1.0))
                cs.box((0.5, -1.0, 0.0), (0.5, 0.25, 1.0))
                cs.sweep((0, 0.5, 0.0), (0.0, -1.5, 0.0), (0, 1, 0), MAX_SLOPE_COS)
            elif kind == "cap":
                if slot + 2 > 96:
                    continue
                cs.agents[1] = [1.4, 0.0, 0.0]
                cs.agents[2] = [1.4, 0.0, 0.0]
                cs.sweep((0, 0, 0), (1.5, 0.0, 0.0))
                first = None
            else:  # inside both at the start: the lower index's separating normal is +x (filtered), the higher one's +y (kept)
                cs.box((-0.5 - 0.1, 0.0, 0.0), (0.5, 2.0, 2.0))
                first = cs.box((0.0, -HH - 0.5 - 0.1, 0.0), (2.0, 0.5, 2.0))  # the winner: the higher index of the pair
                cs.sweep((0, 0, 0), (-0.2, -0.2, 0.0), (0, 1, 0), MAX_SLOPE_COS)
            cs.want = {"tie": kind, "slot": slot}
            if first is not None:
                cs.want["index"] = first
            out.append(cs)
    for slot in (0, 31):  # one lane, two chunks: duplicates at slots j and j + 32, both met at the same fraction
        for axes in (None, yaw_axes(60.0)):
            cs = Case(SWEEP)
            for j in range(slot):
                filler(cs, j)
            first = cs.box((1.2, 0.0, 0.1), (0.1, 0.5, 0.5), axes=axes)
            for j in range(31):
                filler(cs, j)
            cs.box((1.2, 0.0, 0.1), (0.1, 0.5, 0.5), axes=axes)
            cs.sweep((0, 0, 0), (1.5, 0.0, 0.05))
            cs.want = {"tie": "dup", "slot": slot, "index": first}
            out.append(cs)
    return out


def filler(cs, j):
    """a tiny box within the envelope that no sweep of these families reaches"""
    cs.box((-1.5 + 0.03 * (j % 30), 1.6 + 0.1 * (j // 30), 1.0), (0.005, 0.005, 0.005))


def family_boundaries():
    """fractions exactly 1 (the callback's strict < rejects them) and one float32 step either side, a graze of an edge cylinder at
    distance rho and a few steps either side (disc about 0), face hits landing exactly on |q| = H and a step outside it"""
    out = []
    rho = F32(0.33) - F32(0.04)
    end = F32(2.0) - (F32(0.5) + rho)  # from x = 0 the face x = c - (H + rho) of a box at c = 2: t = end / d.x = 1 when d.x = end
    for k in (-1, 0, 1):
        x = end
        for _ in range(abs(k)):
            x = np.nextafter(x, F32(10 if k > 0 else -10))
        cs = Case(SWEEP)
        cs.box((2.0, 0.0, 0.0), (0.5, 0.5, 0.5))
        cs.sweep((0, 0, 0), (float(x), 0.0, 0.0))
        cs.want = {"boundary": "t=1", "k": k}
        out.append(cs)
    for k in range(-2, 3):  # the path along x passes the box's (+y, z-axis) edge cylinder at distance rho: disc = 0 +- rounding
        y = F32(0.5) + F32(HH) + rho
        for _ in range(abs(k)):
            y = np.nextafter(y, F32(10 if k > 0 else -10))
        cs = Case(SWEEP)
        cs.box((1.5, 0.0, 0.0), (0.5, 0.5, 0.5))
        cs.sweep((0.0, float(y), 0.1), (2.0, float(y), 0.1))
        cs.want = {"boundary": "graze", "k": k}
        out.append(cs)
    for k in (0, 1):  # a face hit on the face's border |q_z| = H_z, then one step outside it (the edge takes over)
        z = F32(0.5)
        if k:
            z = np.nextafter(z, F32(10))
        cs = Case(SWEEP)
        cs.box((1.5, 0.0, 0.0), (0.5, 0.5, 0.5))
        cs.sweep((0.0, 0.0, float(z)), (2.0, 0.0, float(z)))
        cs.want = {"boundary": "border", "k": k}
        out.append(cs)
    return out


def family_slope():
    """the slope filter: a closest hit rejected while a farther collider passes, and minSlopeDot at exactly dot(filterDir, n) of an
    edge hit and one float32 step either side (n as the oracle computes it, the decision the filter takes on it)"""
    import orc

    out = []
    cs = Case(SWEEP)
    cs.box((1.0 + RHO + 0.2, -1.0, 0.0), (0.2, 0.3, 1.0))  # a wall, met first along the path, normal -x: filtered
    first = cs.box((0.0, -1.5 - 0.5 - HH - RHO, 0.0), (3.0, 0.5, 3.0))  # a floor whose inflated top is y = -1.5: passes
    cs.sweep((0, 0, 0), (2.0, -2.0, 0.0), (0, 1, 0), MAX_SLOPE_COS)
    cs.want = {"slope": "filtered first", "index": first}
    out.append(cs)
    for yaw in (0.0, 30.0):
        probe = Case(SWEEP)
        axes = yaw_axes(yaw) if yaw else None
        probe.box((1.2, -0.9, 0.0), (0.3, 0.1, 0.3), axes=axes)  # the path meets the box's upper x edge
        probe.sweep((0, 0, 0), (2.0, -0.5, 0.0), (0, 1, 0), -1.0)
        _, of = orc.kcc_cases(*pack([probe]))
        dot = F32(0.0) * F32(of[0, 1]) + F32(1.0) * F32(of[0, 2]) + F32(0.0) * F32(of[0, 3])
        for k in (-1, 0, 1):
            m = dot if k == 0 else np.nextafter(dot, F32(k))
            cs = Case(SWEEP)
            cs.statics = list(probe.statics)
            cs.sweep((0, 0, 0), (2.0, -0.5, 0.0), (0, 1, 0), float(m))
            cs.want = {"slope": "at the threshold", "k": k}
            out.append(cs)
    return out


def family_starts():
    """degenerate paths (d = 0, one or two zero components, 1e-6 and 4 units) and starts inside moving in, out and along, with
    dot(d, n0) at -FLT_EPSILON and one float32 step either side"""
    out = []
    eps = F32(1.1920929e-07)
    for dx in (float(np.nextafter(-eps, F32(-1))), float(-eps), float(np.nextafter(-eps, F32(0)))):
        cs = Case(SWEEP)
        cs.box((-0.5 - RHO + 0.05, 0.0, 0.0), (0.5, 1.0, 1.0))  # the start lies 0.05 inside its +x face
        cs.sweep((0, 0, 0), (dx, 0.0, 0.0))
        cs.want = {"start": "inside"}
        out.append(cs)
    for d in ((0, 0, 0), (1.5, 0, 0), (0, -1.5, 0), (0, 0, 1.5), (1e-6, 0, 0), (4.0, 0.0, 0.0), (1.0, 0.0, 1.0), (-0.3, 0.2, 0.0), (0.0, 0.3, 0.0)):
        for start_inside in (False, True):
            cs = Case(SWEEP)
            off = 0.05 if start_inside else -0.0004
            cs.box((1.0 + 0.5 + RHO - off, 0.0, 0.0), (0.5, 0.5, 0.5))
            cs.box((0.0, -HH - 0.5 - RHO - 0.3, 0.0), (3.0, 0.5, 3.0))
            cs.sweep((1.0, 0, 0), np.array((1.0, 0, 0)) + np.array(d, dtype=np.float64))
            cs.want = {"start": "inside" if start_inside else "outside"}
            out.append(cs)
    # exactly on the rounded face: t = 0 from outside when d0 - rho rounds to > 0, else the inside rule
    for k in range(-2, 3):
        cs = Case(SWEEP)
        x = float(np.float32(0.5 + RHO))
        for _ in range(abs(k)):
            x = float(np.nextafter(F32(x), F32(10 if k > 0 else -10)))
        cs.box((0.0, 0.0, 0.0), (0.5, 0.5, 0.5))
        cs.sweep((x, 0.0, 0.0), (x - 1.0, 0.0, 0.0))
        cs.want = {"start": "surface"}
        out.append(cs)
    return out


def family_capsules():
    """another agent above (standing on its head), below, beside, at the same centre, and around a start inside moving out"""
    out = []
    for name, other, a, b in (
        ("above", (0.0, 2.1, 0.0), (0, 0, 0), (0, 0.5, 0)),
        ("below", (0.0, -2.0, 0.0), (0, 0, 0), (0, -0.6, 0)),
        ("beside", (0.9, 0.0, 0.0), (0, 0, 0), (0.8, 0.0, 0.1)),
        ("same", (0.0, 0.0, 0.0), (0, 0, 0), (0.3, 0.0, 0.0)),
        ("inside_out", (0.2, 0.0, 0.0), (0, 0, 0), (-0.5, 0.0, 0.0)),
        ("inside_in", (0.2, 0.0, 0.0), (0, 0, 0), (0.5, 0.0, 0.0)),
        ("edge", (1.0, 0.1, 0.3), (0, 0, 0), (1.5, -0.4, 0.6)),
    ):
        cs = Case(SWEEP, A=2, agent=0)
        cs.agents[1] = [f32(v) for v in other]
        cs.sweep(a, b, (0, 1, 0) if name == "above" else (0, 0, 0), 0.0 if name == "above" else -1.0)
        cs.want = {"capsule": name}
        out.append(cs)
    return out


def family_recover():
    """depth at -0.041 and a few float32 steps either side, several penetrating colliders across slots 31|32 (the first in collider order
    pushes), the centre of a cube (an axis tie), coincident capsules, rotated boxes"""
    out = []
    for k in range(-3, 4):
        cs = Case(RECOVER)
        x = F32(0.5 + kcc_ref.R - 0.041)
        for _ in range(abs(k)):
            x = np.nextafter(x, F32(10 if k > 0 else -10))
        cs.box((0.0, 0.0, 0.0), (0.5, 0.5, 0.5))
        cs.recover((float(x), 0.0, 0.0))
        cs.want = {"recover": "threshold"}
        out.append(cs)
    for first in (30, 31, 32, 33):
        cs = Case(RECOVER)
        for j in range(40):
            if j < first:
                cs.box((2.0, 1.0 + 0.05 * j, 2.0), (0.01, 0.01, 0.01))
            else:
                cs.box((0.3 + 0.01 * (j - first), 0.0, 0.0), (0.2, 0.2, 0.2))
        cs.recover((0.0, 0.0, 0.0))
        cs.want = {"recover": "first", "index": first}
        out.append(cs)
    for name in ("centre", "capsule", "rot30", "rot60", "rot45"):
        A = 2 if name == "capsule" else 1
        cs = Case(RECOVER, A=A)
        if name == "centre":
            cs.box((0.0, 0.0, 0.0), (1.0, 1.0 - HH, 1.0))
        elif name == "capsule":
            cs.agents[1] = [0.0, 0.0, 0.0]
        else:
            cs.box((0.35, 0.1, 0.05), (0.3, 0.5, 0.05), axes=yaw_axes(float(name[3:])))
        cs.recover((0.0, 0.0, 0.0))
        cs.want = {"recover": name}
        out.append(cs)
    return out


def family_steps(seed=3):
    """controller steps: ledges just below and above the step height, two- and three-box corners, grazing slides and rotated maze-wall
    junctions, a jump into a ceiling, a fall at the 55 u/s cap onto thin boxes and seams, standing on another agent, embedded in large
    boxes, horizontal speeds up to 60 u/s, colliders 2.8 to 3.2 from the agent"""
    rng = np.random.default_rng(seed)
    out = []
    floor_y = -HH - kcc_ref.R - 0.5  # a floor whose top the standing capsule rests on

    def floor(cs, x=0.0, z=0.0, half=6.0):
        cs.box((x, floor_y, z), (half, 0.5, half))

    for h in (0.15, 0.19, 0.2, 0.21, 0.25, 0.4):  # a ledge just below and just above the climbable height
        for sp in (2.0, 4.5):
            cs = Case(STEP)
            floor(cs)
            cs.box((1.0, floor_y + 0.5 + h - 0.5, 0.0), (0.5, 0.5, 2.0))
            cs.step((0.0, 0.0, 0.0), hvel=(sp * 15 * 0.1, 0, 0), vvel=0.0)
            cs.want = {"step": "ledge"}
            out.append(cs)
    for yaw in (0.0, 30.0, 60.0, 45.0):  # concave corners of two and three boxes, pushed into at speed
        for n in (2, 3):
            cs = Case(STEP)
            floor(cs)
            ax = yaw_axes(yaw) if yaw else None
            cs.box(_to_world(ax, (0.9, 0.5, 0.0)), (0.2, 1.5, 2.0), axes=ax)
            cs.box(_to_world(ax, (0.0, 0.5, 0.9)), (2.0, 1.5, 0.2), axes=ax)
            if n == 3:
                cs.box(_to_world(ax, (0.0, 1.4, 0.0)), (2.0, 0.2, 2.0), axes=ax)
            v = _to_world(ax, (20.0, 0.0, 20.0))
            cs.step((0.0, 0.0, 0.0), hvel=v)
            cs.want = {"step": "corner"}
            out.append(cs)
    for ang in (0.0, 1e-3, 0.01, 0.3):  # grazing slides along a wall
        cs = Case(STEP)
        floor(cs)
        cs.box((0.0, 0.5, 0.5 + RHO + 0.3 - 1e-4), (4.0, 1.5, 0.3))
        cs.step((0.0, 0.0, 0.0), hvel=(4.5 * math.cos(ang), 0, 4.5 * math.sin(ang)))
        cs.want = {"step": "graze"}
        out.append(cs)
    for k in range(3):  # rotated maze-wall junctions (hex walls meet at 120 degrees)
        cs = Case(STEP)
        floor(cs)
        for yaw in (0.0 + 60 * k, 120.0 + 60 * k, 240.0 + 60 * k):
            ax = yaw_axes(yaw)
            cs.box(_to_world(ax, (1.2, 0.5, 0.0)), (1.0, 1.5, 0.1), axes=ax)
        v = _to_world(yaw_axes(60 * k + 10), (8.0, 0.0, 0.0))
        cs.step((0.0, 0.0, 0.0), hvel=v)
        cs.want = {"step": "junction"}
        out.append(cs)
    for gap in (0.05, 0.3, 0.6):  # a jump into a ceiling
        cs = Case(STEP)
        floor(cs)
        cs.box((0.0, HH + kcc_ref.R + gap + 0.25, 0.0), (2.0, 0.25, 2.0))
        cs.step((0.0, 0.0, 0.0), vvel=6.2, jump_speed=6.2, was_jumping=True)
        cs.want = {"step": "ceiling"}
        out.append(cs)
    for top in (0.5, 2.0, 3.5):  # a fall at the 55 u/s cap onto thin boxes and a seam
        for seam in (False, True):
            cs = Case(STEP)
            ytop = -HH - kcc_ref.R - top
            if seam:
                cs.box((-0.5, ytop - 0.01, 0.0), (0.5, 0.01, 1.0))
                cs.box((0.5, ytop - 0.01, 0.0), (0.5, 0.01, 1.0))
            else:
                cs.box((0.0, ytop - 0.005, 0.0), (1.0, 0.005, 1.0))
            cs.step((0.0, 0.0, 0.0), vvel=-55.0, voff=-55.0 * DT)
            cs.want = {"step": "fall"}
            out.append(cs)
    for dx in (0.0, 0.2, 0.5):  # standing on another agent
        cs = Case(STEP, A=2, agent=0)
        floor(cs)
        cs.agents[1] = [dx, 0.0, 0.0]
        cs.step((0.0, 2 * HH + 2 * kcc_ref.R + 0.05, 0.0), vvel=-1.0)
        cs.want = {"step": "on_agent"}
        out.append(cs)
    for depth in (0.3, 1.0, 2.5):  # embedded in large boxes: push-outs, then speed left over
        cs = Case(STEP)
        floor(cs)
        cs.box((depth - 3.0, 0.0, 0.0), (3.0, 3.0, 3.0))
        cs.step((0.0, 0.0, 0.0), hvel=(0.0, 0.0, 0.0))
        cs.want = {"step": "embedded"}
        out.append(cs)
    for sp in (10.0, 30.0, 45.0, 60.0):  # fast states, walls at the envelope's edge
        for dist in (2.8, 2.9, 3.0, 3.1, 3.2):
            cs = Case(STEP)
            floor(cs)
            cs.box((dist + 0.2, 0.5, 0.0), (0.2, 1.5, 2.0))
            th = rng.uniform(-0.3, 0.3)
            cs.step((0.0, 0.0, 0.0), hvel=(sp * math.cos(th), 0.0, sp * math.sin(th)))
            cs.want = {"step": "edge"}
            out.append(cs)
    return out


def hunt_steps(n, seed):
    """random controller states and colliders around the envelope's edge (fast states, boxes 2.5 to 3.6 away, agents anywhere near)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        A = int(rng.integers(1, 4))
        cs = Case(STEP, A=A, agent=0)
        cs.box((0.0, -HH - kcc_ref.R - 0.5 + rng.uniform(-0.1, 0.05), 0.0), (8.0, 0.5, 8.0))
        for _ in range(int(rng.integers(1, 12))):
            r = rng.uniform(2.5, 3.6)
            th = rng.uniform(0, 2 * math.pi)
            ax = yaw_axes(float(rng.choice(YAWS))) if rng.random() < 0.4 else None
            cs.box((r * math.cos(th), rng.uniform(-1.5, 1.5), r * math.sin(th)), rng.uniform(0.05, 1.5, 3), axes=ax)
        for a in range(1, A):
            cs.agents[a] = [f32(v) for v in rng.uniform(-3.5, 3.5, 3) * (1, 0.3, 1)]
        sp = rng.uniform(0, 60)
        th = rng.uniform(0, 2 * math.pi)
        vv = float(rng.choice([0.0, -55.0, 6.2, rng.uniform(-55, 6.2)]))
        cs.step((0.0, rng.uniform(-0.2, 0.2), 0.0), hvel=(sp * math.cos(th), 0.0, sp * math.sin(th)), vvel=vv, voff=vv * DT,
                jump_speed=6.2, was_jumping=bool(vv > 0))
        cs.want = {"step": "hunt"}
        out.append(cs)
    return out


def family_envelope():
    """one box or one other agent just inside and just outside each of the six faces of the culling envelope (x and z +-3, y -6 / +3
    round the agent): its bounds grown by the capsule overlap the envelope by 0.01, or miss it by 0.01"""
    out = []
    pos = np.array([0.3, 0.2, -0.4])
    lo, hi = pos - (3.0, 6.0, 3.0), pos + (3.0, 3.0, 3.0)
    R = kcc_ref.R
    for kind in ("box", "cap"):
        ext = np.array([0.2 + R, 0.2 + HH + R, 0.2 + R]) if kind == "box" else np.array([2 * R + 3, 2 * (HH + R) + 6, 2 * R + 3])
        for axis in range(3):
            for side in (-1, 1):
                for gap in (-0.01, 0.01):
                    c = pos.copy()
                    c[axis] = (hi[axis] + gap + ext[axis]) if side > 0 else (lo[axis] - gap - ext[axis])
                    cs = Case(SWEEP, A=2 if kind == "cap" else 1, pos=pos)
                    if kind == "box":
                        cs.box(c, (0.2, 0.2, 0.2))
                    else:
                        cs.agents[1] = [f32(v) for v in c]
                    cs.sweep(pos, pos + (0.1, 0.0, 0.0))
                    cs.want = {"envelope": (kind, axis, side), "candidates": int(gap < 0)}
                    out.append(cs)
    return out


SWEEP_FAMILIES = {"features": family_features, "decode": family_decode, "counts": family_counts, "ties": family_ties,
                  "starts": family_starts, "capsules": family_capsules, "boundaries": family_boundaries, "slope": family_slope}
