"""Constructed scene families for the rasteriser: each puts triangles where a rasteriser's branches and thresholds are (test
infrastructure).  A scene is (view16, instances): one camera at the origin looking down -z (identity view), instances as rows of 18
floats (mesh, colour, 16 model floats column-major), sorted by mesh type as the product's instance lists are.  Every family is built
for any frame size W x H, and check_reach(family, render) says whether the reference's record shows that the scene reached what the
family is for -- so a scene that drifts away from its branch fails instead of passing vacuously."""
import numpy as np

import raster_ref as ref

F32 = np.float32
IDENTITY = np.eye(4, dtype=F32).reshape(-1)


def _row(mesh, color, m):
    return np.concatenate([[mesh, color], np.asarray(m, dtype=np.float64).T.reshape(-1)])


def _model(center, half, rot=None):
    m = np.eye(4)
    m[:3, :3] = (np.eye(3) if rot is None else rot) @ np.diag(half)
    m[:3, 3] = center
    return m


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])


def _view_xy(px, py, depth, W, H):
    """view-space x, y of the point at distance `depth` in front of the camera that projects onto window position (px, py), in pixels"""
    p00, p11, _, _ = ref.projection(W, H)
    return (px - W / 2) / (W / 2) * depth / float(p00), (py - H / 2) / (H / 2) * depth / float(p11)


def _scene(rows):
    rows = sorted(rows, key=lambda r: r[0])  # stable: draw order within a mesh type is the order given
    return IDENTITY.copy(), np.array(rows, dtype=F32)


def _pixel_box(px0, py0, px1, py1, z_front, half_z, W, H, color):
    """a box whose front face covers the window rectangle with corners on the pixel CENTRES (px0 + .5, py0 + .5) .. (px1 + .5, py1 + .5)"""
    return _window_box(px0 + 0.5, py0 + 0.5, px1 + 0.5, py1 + 0.5, z_front, half_z, W, H, color)


def _window_box(wx0, wy0, wx1, wy1, z_front, half_z, W, H, color):
    """a box whose front face covers the window rectangle (wx0, wy0) .. (wx1, wy1), in pixels"""
    (x0, y0), (x1, y1) = _view_xy(wx0, wy0, -z_front, W, H), _view_xy(wx1, wy1, -z_front, W, H)
    return _row(0, color, _model([(x0 + x1) / 2, (y0 + y1) / 2, z_front - half_z], [abs(x1 - x0) / 2, abs(y1 - y0) / 2, half_z]))


def far_plane(W, H, seed=0):
    """boxes straddling the far plane (z = -120), one wholly beyond it, and long boxes from behind the camera to beyond the far plane,
    whose side faces are cut by both planes (five-sided polygons)"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(4):
        x, y = _view_xy(rng.uniform(0.2, 0.8) * W, rng.uniform(0.2, 0.8) * H, 118.0, W, H)
        rows.append(_row(0, k, _model([x, y, -119.0 - rng.uniform(-1, 1)], [rng.uniform(5, 25), rng.uniform(5, 15), 4.0], _rot(*rng.uniform(-0.4, 0.4, 3)))))
    rows.append(_row(0, 5, _model([0, 0, -140.0], [30, 30, 5])))  # wholly beyond the far plane
    for k in range(4):  # sheared slabs: face corners at depths of about +40, -20, -100 and -160, so that both planes cut a triangle
        m = np.eye(4)
        m[:3, 0] = [0.2, 0, 0]
        m[:3, 1] = [0, rng.uniform(1, 3), -30.0] if k % 2 else [rng.uniform(1, 3), 0, -30.0]
        m[:3, 2] = [rng.uniform(-1, 1), rng.uniform(-1, 1), -70.0]
        m[:3, 3] = [(-1) ** k * rng.uniform(0.5, 2.0), rng.uniform(-1, 1), -60.0]
        rows.append(_row(0, 6 + k, m))
    rows.append(_row(2, 9, _model([0, 0, -120.0], [6, 6, 6])))  # a sphere through the far plane
    return _scene(rows)


def edge_bounds(W, H, seed=0):
    """screen-facing boxes from a tenth of the frame to several frames across: their triangles' edge bounds straddle 2^30"""
    rng = np.random.default_rng(seed)
    rows = []
    s0 = 2.0 ** 14 / (1.5 * (W + H))  # pixels across at which the bound (about 1.5 * 256^2 * size * (W + H)) is 2^30
    for k in range(24):
        size = s0 * np.exp(rng.uniform(np.log(0.25), np.log(4.0)))
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        z = rng.uniform(2.0, 20.0)
        (x0, y0), (x1, y1) = _view_xy(cx - size / 2, cy - size * rng.uniform(0.3, 1.0) / 2, z, W, H), _view_xy(cx + size / 2, cy + size / 2, z, W, H)
        rows.append(_row(0, k % 20, _model([(x0 + x1) / 2, (y0 + y1) / 2, -z - 0.5], [abs(x1 - x0) / 2, abs(y1 - y0) / 2, 0.5], _rot(0, 0, rng.uniform(-0.5, 0.5)))))
    return _scene(rows)


def tiny_and_large(W, H, seed=0):
    """many triangles of a few pixels (a rasteriser's one-lane path), some with corners on the pixel centres at tile corners, over and
    under large ones"""
    rng = np.random.default_rng(seed)
    rows = [_row(0, 0, _model(list(_view_xy(W * 0.5, H * 0.5, 30.0, W, H)) + [-30.0], [30.0 * W / 100, 30.0 * H / 100, 1.0], _rot(0, 0, 0.3)))]
    for k in range(60):  # tiny boxes and spheres, slightly rotated
        z = rng.uniform(5.0, 29.0)
        x, y = _view_xy(rng.uniform(0, W), rng.uniform(0, H), z, W, H)
        s = z * rng.uniform(0.3, 2.0) / W
        rows.append(_row(int(rng.choice([0, 0, 2, 3])), k % 20, _model([x, y, -z], [s, s * rng.uniform(0.5, 2), s], _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    for tx in range(32, W, 32):  # 1..2-pixel boxes with corners on the pixel centres around tile corners
        for ty in range(4, H, 4 * max(1, H // 16)):
            w_, h_ = int(rng.integers(1, 3)), int(rng.integers(1, 3))
            rows.append(_pixel_box(tx - w_, ty - h_, tx, ty, -rng.uniform(3.0, 20.0), 0.05, W, H, int(rng.integers(0, 20))))
    rows.append(_row(4, 3, _model([0, 0, -3.0], [0.4, 0.4, 0.4], _rot(0.5, 0.2, 0))))  # and a large cylinder over them
    return _scene(rows)


def duplicates(W, H, seed=0, gap=0, count=24):
    """coincident duplicate instances in different colours: instance j and j + gap (gap 0: the copy follows directly) are the same box or
    mesh, so every pixel of the pair is a depth tie that the later draw must win.  gap > 128 puts the copies in different 128-instance
    chunks of the rasteriser; filler boxes far away keep the copies apart in the list"""
    rng = np.random.default_rng(seed)
    base = []
    for k in range(count):
        z = rng.uniform(3.0, 15.0)
        x, y = _view_xy(rng.uniform(0, W), rng.uniform(0, H), z, W, H)
        base.append((0 if k < count * 2 // 3 else int(rng.integers(1, 5)), _model([x, y, -z], rng.uniform(0.3, 1.5, 3), _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    boxes = [b for b in base if b[0] == 0]
    meshes = [b for b in base if b[0] != 0]
    rows = []
    if gap == 0:
        for mesh, m in boxes + meshes:
            rows += [_row(mesh, int(rng.integers(0, 10)), m), _row(mesh, int(rng.integers(10, 20)), m)]
        return _scene(rows)
    assert gap >= len(boxes)
    filler = [_row(0, 21, _model([rng.uniform(-50, 50), rng.uniform(-30, 30), -100.0], [0.2, 0.2, 0.2])) for _ in range(gap - len(boxes))]
    rows = [_row(0, int(rng.integers(0, 10)), m) for _, m in boxes] + filler + [_row(0, int(rng.integers(10, 20)), m) for _, m in boxes]
    rows += [r for mesh, m in meshes for r in (_row(mesh, 3, m), _row(mesh, 13, m))]
    return _scene(rows)


def mirrored(W, H, seed=0):
    """boxes and meshes under transforms with one or three negative scales (mirroring: the winding turns round) and with two (a rotation)"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(12):
        z = rng.uniform(3.0, 9.0)
        x, y = _view_xy(rng.uniform(0.1, 0.9) * W, rng.uniform(0.1, 0.9) * H, z, W, H)
        sign = [[-1, 1, 1], [1, -1, 1], [1, 1, -1], [-1, -1, -1], [-1, -1, 1]][k % 5]
        mesh = 0 if k < 7 else int(rng.integers(1, 5))
        rows.append(_row(mesh, k, _model([x, y, -z], np.array(sign) * rng.uniform(0.4, 1.2, 3), _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    return _scene(rows)


def grazing(W, H, seed=0):
    """faces seen at about 0.02 rad (a rasteriser's object-space and box-face tests decide near there) under per-axis scales from 1e-3
    to 1e3: boxes turned until a face's plane almost contains the eye, and stretched spheres and cylinders"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(16):
        z = rng.uniform(3.0, 12.0)
        x, y = _view_xy(rng.uniform(0.15, 0.85) * W, rng.uniform(0.15, 0.85) * H, z, W, H)
        c = np.array([x, y, -z])
        half = np.array([10.0 ** rng.uniform(-3, 0.3), 10.0 ** rng.uniform(-3, 0.3), 10.0 ** rng.uniform(-3, 0.3)])
        half[k % 3] = 10.0 ** rng.uniform(-3, -1)  # a thin axis: the face across it is large, the others small
        # turn the box so that the plane of face +axis makes the angle ang with the direction from its centre to the eye
        d = -c / np.linalg.norm(c)
        ang = rng.choice([-1, 1]) * rng.uniform(0.005, 0.04)
        side = np.cross(d, [0.3, 1.0, 0.1]); side /= np.linalg.norm(side)
        n = np.cos(ang) * side + np.sin(ang) * d  # unit normal of the face, at angle ang to the plane through the eye
        u = np.cross(n, [0.7, 0.2, 0.5]); u /= np.linalg.norm(u)
        v = np.cross(n, u)
        axis = k % 3
        R = np.zeros((3, 3)); R[:, axis] = n; R[:, (axis + 1) % 3] = u; R[:, (axis + 2) % 3] = v
        if np.linalg.det(R) < 0:
            R[:, (axis + 2) % 3] *= -1
        rows.append(_row(0, k % 20, _model(c - n * half[axis], half, R)))  # the face's centre sits at c
    for k in range(6):
        z = rng.uniform(3.0, 12.0)
        x, y = _view_xy(rng.uniform(0.2, 0.8) * W, rng.uniform(0.2, 0.8) * H, z, W, H)
        half = np.array([10.0 ** rng.uniform(-3, 3) for _ in range(3)]).clip(1e-3, 30.0)
        rows.append(_row(int(rng.choice([2, 4])), k, _model([x, y, -z - float(half.max())], half, _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    return _scene(rows)


def frustum_tangent(W, H, seed=0):
    """spheres and boxes just outside a side plane of the view frustum, reaching a little way in: the instance-level frustum test has to
    keep them (its bounding sphere is conservative, the meshes are within a few per cent of the tangent position)"""
    rng = np.random.default_rng(seed)
    p00, p11, _, _ = ref.projection(W, H)
    rows = []
    for k in range(16):
        z = rng.uniform(2.0, 10.0)
        r = rng.uniform(0.2, 0.8)
        mesh = 2 if k % 2 else 0
        rad = r if mesh == 2 else r * np.sqrt(3.0)   # the true bounding radius (the rasteriser's conservative bound is larger)
        eps = -rng.uniform(0.1, 0.3) * rad  # the mesh reaches a little way into the frustum: a sliver at the frame's edge
        side = k % 4
        # side planes x = +-w / p00, y = +-w / |p11|: put the centre at distance rad + eps outside the plane (inward normal)
        ax = float(abs(p00)) if side < 2 else float(abs(p11))
        t = (z * 1.0 + (rad + eps) * np.sqrt(ax * ax + 1.0)) / ax  # |x| * ax - z = (rad + eps) * sqrt(ax^2 + 1)
        pos = [0.0, 0.0, -z]
        pos[0 if side < 2 else 1] = t if side % 2 == 0 else -t
        rows.append(_row(mesh, k % 20, _model(pos, [r, r, r], None if mesh == 2 else _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    return _scene(rows)


def slivers(W, H, seed=0):
    """degenerate and nearly degenerate triangles: boxes squashed to zero extent along an axis (faces of zero area), boxes one sub-pixel
    wide across pixel centres, and needle triangles"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(8):
        z = rng.uniform(3.0, 10.0)
        x, y = _view_xy(rng.uniform(0.1, 0.9) * W, rng.uniform(0.1, 0.9) * H, z, W, H)
        half = rng.uniform(0.3, 1.0, 3)
        half[k % 3] = 1e-7 if k < 4 else 1e-4
        rows.append(_row(0, k, _model([x, y, -z], half, _rot(*rng.uniform(0, 0.2, 3)))))
    for k in range(10):  # one or two sub-pixels wide, across a column of pixel centres
        z = rng.uniform(3.0, 10.0)
        px, py = int(rng.integers(2, W - 2)), int(rng.integers(2, H - 8))
        (x0, y0), (x1, y1) = _view_xy(px + 0.5 - (k % 2 + 1) / 512, py + 0.5, z, W, H), _view_xy(px + 0.5 + (k % 2 + 1) / 512, py + 6.5, z, W, H)
        rows.append(_row(0, 10 + k, _model([(x0 + x1) / 2, (y0 + y1) / 2, -z - 0.1], [abs(x1 - x0) / 2, abs(y1 - y0) / 2, 0.1], _rot(0, 0, 0.02 * (k - 5)))))
    return _scene(rows)


def borders(W, H, seed=0, band_rows=()):
    """box edges on the pixel centres of the viewport's last column and last row, of its first ones, and of the rows either side of band
    boundaries"""
    rng = np.random.default_rng(seed)
    rows = []
    z = lambda: -rng.uniform(3.0, 9.0)
    rows.append(_pixel_box(W - 9, 3, W - 1, min(H - 1, 12), z(), 0.3, W, H, 1))      # right edge on the last column's centres
    rows.append(_pixel_box(3, H - 4, min(W - 1, 20), H - 1, z(), 0.3, W, H, 2))      # bottom edge on the last row's centres
    rows.append(_window_box(W - 5.5, H - 3.5, W, H, z(), 0.3, W, H, 3))              # right and bottom edges on the viewport's border
    rows.append(_window_box(W / 2 + 0.5, H / 2 + 0.5, W + 0.5, H + 0.5, z(), 0.3, W, H, 7))  # ... and half a pixel beyond it
    rows.append(_pixel_box(0, 0, 6, 3, z(), 0.3, W, H, 4))
    for k, r in enumerate(band_rows):
        if 0 < r < H:
            x0 = int(rng.integers(0, max(1, W - 12)))
            rows.append(_pixel_box(x0, r - 2, x0 + 9, r - 1, z(), 0.2, W, H, 5 + k % 10))  # ends on the band's last row
            rows.append(_pixel_box(x0 + 3, r, x0 + 12 if x0 + 12 < W else W - 1, r + 1, z(), 0.2, W, H, 6 + k % 10))  # starts on the next band's first
    return _scene(rows)


def ties(W, H, seed=0):
    """screen-facing boxes whose front-face corners project onto pixel centres: whole rows and columns of samples and the face diagonals
    lie exactly on edges"""
    rng = np.random.default_rng(3000 + seed)
    rows = []
    for k in range(6):
        z_front = -rng.uniform(3.0, 9.0)
        wpx = int(rng.integers(6, max(8, W // 4))); hpx = wpx if k % 2 == 0 else int(rng.integers(6, max(8, H // 3)))
        wpx, hpx = min(wpx, W - 2), min(hpx, H - 2)
        px0, py0 = int(rng.integers(0, W - wpx)), int(rng.integers(0, H - hpx))
        rows.append(_pixel_box(px0, py0, px0 + wpx, py0 + hpx, z_front, rng.uniform(0.2, 0.6), W, H, k))
    return _scene(rows)


def offscreen_vertex(W, H, log2_px, opposite=False):
    """screen-facing triangles (thin boxes) with one corner 2^log2_px pixels beyond the right edge of the frame, just in front of the
    near plane (w = 0.02), the others on screen; opposite: the box spans from 2^log2_px pixels left of the frame to as far right of it"""
    rows = []
    for k, (py, w) in enumerate(((H * 0.3, 0.02), (H * 0.6, 0.05))):
        far_x = _view_xy(W + 2.0 ** log2_px, py, w, W, H)[0]
        near_x = _view_xy(-(2.0 ** log2_px), py, w, W, H)[0] if opposite else _view_xy(W * 0.25, py, w, W, H)[0]
        y0, y1 = _view_xy(0, py - H * 0.15, w, W, H)[1], _view_xy(0, py + H * 0.15, w, W, H)[1]
        m = np.eye(4)
        m[:3, 0] = [(far_x - near_x) / 2, 0, 0]
        m[:3, 1] = [0.1 * (far_x - near_x) / 2 * (k - 0.5), (y1 - y0) / 2, 0]  # sheared: the edges to the far corner are slanted
        m[:3, 2] = [0, 0, w * 0.001]
        m[:3, 3] = [(far_x + near_x) / 2, (y0 + y1) / 2, -w - w * 0.001]
        rows.append(_row(0, k, m))
    return _scene(rows)


def _unit(v):
    return np.asarray(v, dtype=np.float64) / np.linalg.norm(v)


def _basis(axis_dir, axis, hint=(0.3, 0.9, 0.2)):
    """a rotation whose column `axis` is the unit vector axis_dir"""
    n = _unit(axis_dir)
    u = _unit(np.cross(n, hint))
    R = np.zeros((3, 3))
    R[:, axis], R[:, (axis + 1) % 3], R[:, (axis + 2) % 3] = n, u, np.cross(n, u)
    return R


def _cells(n, W, H, max_aspect=None):
    """centres (px, py) and size in pixels of n cells of a grid laid over the frame with about square cells; max_aspect: over the central
    part of the frame at most that many times wider than high or higher than wide"""
    w, h = (W, H) if max_aspect is None else (min(W, max_aspect * H), min(H, max_aspect * W))
    cols = max(1, min(n, int(round(np.sqrt(n * w / h)))))
    rows = -(-n // cols)
    cw, ch = w / cols, h / rows
    return [((W - w) / 2 + (k % cols + 0.5) * cw, (H - h) / 2 + (k // cols + 0.5) * ch) for k in range(n)], min(cw, ch)


def _px_size(z, W, H):
    """view-space length of one pixel at distance z (pixels are square)"""
    p00, _, _, _ = ref.projection(W, H)
    return z / (float(p00) * W / 2)


def _bisector(c):
    """unit normal that reflects the light at point c (view space) into the eye: the bisector of the directions to the light and the eye"""
    return _unit(_unit(ref.LIGHT - c) + _unit(-c))


def highlights(W, H, seed=0):
    """spheres, capsules, cylinders and boxes turned so that the light's reflection reaches the eye: box faces and curved sides whose
    normal is the bisector of the light and eye directions -- highlights that saturate, and the fall-off around them through the fast
    fragment stage's vdr cut-off (0.97)"""
    rng = np.random.default_rng(seed)
    kinds = [0, 2, 0, 1, 4, 0, 2, 4, 0, 1, 3, 2]
    centres, cell = _cells(len(kinds), W, H)
    rows = []
    for k, (mesh, (px, py)) in enumerate(zip(kinds, centres)):
        z = rng.uniform(3.0, 8.0)
        c = np.array(list(_view_xy(px, py, z, W, H)) + [-z])
        r = 0.42 * cell * _px_size(z, W, H)
        b = _bisector(c)
        if mesh == 0:  # face +z across the bisector, its centre at c
            R = _basis(b, 2)
            half = np.array([r, r * rng.uniform(0.6, 1.0), 0.3 * r])
            rows.append(_row(0, k % 22, _model(c - b * half[2], half, R)))
        elif mesh == 2:
            rows.append(_row(2, k % 22, _model(c - b * r, [r, r, r], _rot(*rng.uniform(0, 2 * np.pi, 3)))))
        else:  # capsule, cone, cylinder: axis (y) across the bisector, so that a line of the side faces it
            R = _basis(b, 0)
            ry = r * (0.5 if mesh == 1 else 1.0)
            rows.append(_row(mesh, k % 22, _model(c - b * 0.6 * r, [0.6 * r, ry, 0.6 * r], R)))
    return _scene(rows)


def light_gates(W, H, seed=0):
    """box faces in planes that pass the light at a chosen signed distance: N.L = delta / |light - P| over the whole face, so a face lies
    wholly at intensity 0, inside (0, 0.001] (the highlight is gated off), or just above 0.001 (it is computed)"""
    rng = np.random.default_rng(seed)
    targets = [-0.05, 0.0, 0.0005, 0.0008, 0.0013, 0.002, -0.0005, 0.0006, 0.0016]
    centres, cell = _cells(len(targets), W, H, max_aspect=2)  # (at the far ends of a 16:1 frame the eye and light directions nearly meet)
    rows = []
    for k, (t, (px, py)) in enumerate(zip(targets, centres)):
        z = rng.uniform(3.0, 8.0)
        c = np.array(list(_view_xy(px, py, z, W, H)) + [-z])
        L, V = _unit(ref.LIGHT - c), _unit(-c)
        perp = _unit(V - V.dot(L) * L)   # in the plane through the light, as near the eye direction as it gets
        n = np.sqrt(1.0 - t * t) * perp + t * L   # N.(light - c) = t |light - c|: the plane passes the light at distance t |light - c|
        r = 0.45 * cell * _px_size(z, W, H) / max(0.3, n.dot(V))  # the face is seen obliquely: stretch it to fill the cell
        half = np.array([r, r, 0.2 * r])
        rows.append(_row(0, k % 22, _model(c - n * half[2], half, _basis(n, 2, hint=np.cross(n, V) + 0.01))))
    return _scene(rows)


def scaled_normals(W, H, seed=0):
    """spheres, capsules, cones, cylinders and boxes under rotations with per-axis scales from 1e-2 to 1e2 of a common size (ratios up to
    1e4), some mirrored: the normal matrix (inverse transpose) and the model matrix turn the normals far apart"""
    rng = np.random.default_rng(seed)
    kinds = [2, 1, 3, 4, 2, 0, 2, 4, 3, 1, 2, 0]
    centres, cell = _cells(len(kinds), W, H)
    rows = []
    for k, (mesh, (px, py)) in enumerate(zip(kinds, centres)):
        z = rng.uniform(4.0, 10.0)
        c = np.array(list(_view_xy(px, py, z, W, H)) + [-z])
        u = np.zeros(3)
        u[k % 3], u[(k + 1) % 3], u[(k + 2) % 3] = 2.0, rng.uniform(1.0, 2.0), -2.0  # one axis long, one thin: plates
        s = 10.0 ** u
        s *= 0.45 * cell * _px_size(z, W, H) / s.max()
        if k % 3 == 2:
            s[k % 3] *= -1  # mirrored
        if k % 6 == 5:
            s[:] *= -1      # mirrored along all three axes
        rows.append(_row(mesh, k % 22, _model(c, s, _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    return _scene(rows)


def near_plane(W, H, seed=0):
    """boxes, rods and spheres from behind the camera to in front of it: the near plane cuts flat faces and curved sides (the clipper
    makes vertices whose position and normal are interpolated), to the left, right, above and below the eye and straight ahead"""
    rng = np.random.default_rng(seed)
    rows = [_row(0, 8, _model([0.0, -1.2, -4.0], [3.0, 0.4, 6.0], _rot(0.05, 0.1, 0.0))),   # a floor slab under the camera
            _row(0, 9, _model([1.0, 0.0, -2.0], [0.2, 0.6, 4.0], _rot(0.0, -0.1, 0.05)))]     # and a wall beside it
    for k, (x, y) in enumerate(((0.5, 0.0), (-0.55, 0.05), (0.0, 0.4), (0.05, -0.45))):
        rot = _basis([0.1 * x, 0.1 * y, 1.0], 1)   # cylinder / capsule axis (y) along the view direction
        r = rng.uniform(0.15, 0.25)
        rows.append(_row(4 if k % 2 == 0 else 1, 1 + k, _model([x, y, -1.0], [r, 2.0 if k % 2 == 0 else 1.0, r], rot)))
    for k, (x, y) in enumerate(((0.6, -0.3), (-0.5, 0.3))):
        rows.append(_row(2, 6 + k, _model([x, y, 0.0], [0.45, 0.45, 0.45], _rot(*rng.uniform(0, 2 * np.pi, 3)))))
    rows.append(_row(3, 11, _model([0.0, 0.0, -0.3], [0.08, 0.5, 0.08], _basis([0.05, 0.02, 1.0], 1))))  # a cone pointing at the eye
    return _scene(rows)


def palette(W, H, seed=0):
    """the 22 colours of the palette on boxes facing the camera, lit by the light above and behind it"""
    rng = np.random.default_rng(seed)
    centres, cell = _cells(22, W, H, max_aspect=4)
    rows = []
    for k, (px, py) in enumerate(centres):
        z = rng.uniform(3.0, 8.0)
        h = 0.42 * cell
        rows.append(_window_box(px - h, py - h, px + h, py + h, -z, 0.3, W, H, k))
    return _scene(rows)


FAMILIES = {"far_plane": far_plane, "edge_bounds": edge_bounds, "tiny_and_large": tiny_and_large, "duplicates": duplicates, "mirrored": mirrored,
            "grazing": grazing, "frustum_tangent": frustum_tangent, "slivers": slivers, "borders": borders, "ties": ties,
            "highlights": highlights, "light_gates": light_gates, "scaled_normals": scaled_normals, "near_plane": near_plane, "palette": palette}
CLIPPED = {"far_plane", "near_plane"}  # families whose triangles the clipper cuts (new vertices: a few pixels may differ)


def build(family, W, H, seed=0, **kw):
    return FAMILIES[family](W, H, seed, **kw)


def check_reach(family, R, W, H):
    """assert that the reference's record of the scene shows the branches the family was built for"""
    front = [t for t in R.tris if t["front"] and t["covered"]]
    if family == "far_plane":
        assert R.reached("clip", "far") >= 4, "triangles cut by the far plane"
        assert R.reached("clip", "both") >= 2 and any(t.get("poly") == 5 for t in R.tris), "triangles cut by both planes into five-gons"
        assert R.reached("beyond_far") >= 6, "triangles wholly beyond the far plane"
        assert (R.z[R.inst > 0] > 0.999).any(), "fragments at the far end of the depth range"
    elif family == "edge_bounds":
        bounds = np.array([t["bound"] for t in front], dtype=np.float64)
        assert ((bounds < ref.EDGE_INT32) & (bounds >= ref.EDGE_INT32 / 4)).sum() >= 2, "edge bounds just below 2^30"
        assert ((bounds >= ref.EDGE_INT32) & (bounds < ref.EDGE_INT32 * 4)).sum() >= 2, "edge bounds just above 2^30"
    elif family == "tiny_and_large":
        assert sum(1 for t in front if t["small"]) >= 20, "triangles of at most four pixels of a tile"
        assert sum(1 for t in front if not t["small"]) >= 2
        assert R.ties > 0 or W <= 32, "samples on edges (at tile corners inside the frame)"
    elif family == "duplicates":
        pairs = R.inst[R.inst > 0]
        assert pairs.size > 50
    elif family == "mirrored":
        assert sum(1 for t in front if t["mirrored"]) >= 10, "front faces of mirrored instances drawn"
    elif family == "grazing":
        sines = np.array([t["sin"] for t in R.tris if t["sin"] is not None and not t["culled"]])
        assert ((sines > 0.005) & (sines < 0.04)).sum() >= 4, "front faces seen at about 0.02 rad"
        assert sum(1 for t in R.tris if t["culled"] and t["sin"] is not None and t["sin"] < 0.04) >= 4, "back faces seen at about 0.02 rad"
    elif family == "frustum_tangent":
        assert (R.inst[:, 0] > 0).any() or (R.inst[:, -1] > 0).any() or (R.inst[0] > 0).any() or (R.inst[-1] > 0).any(), "an instance at the frame's edge"
    elif family == "slivers":
        assert R.reached("culled") >= 8, "degenerate triangles"
        assert any(t["min_extent"] <= 2 for t in front), "a triangle at most two sub-pixels wide that covers a sample"
    elif family in ("borders", "ties"):
        assert R.ties > 50, "samples on edges"
        if family == "borders":
            assert (R.inst[:, W - 1] > 0).any() and (R.inst[H - 1] > 0).any(), "the last column and row drawn"
    elif family == "highlights":
        F, drawn = R.frag, R.inst > 0
        vdr = np.nan_to_num(F.vdr, nan=-1.0)
        flat = np.array([t["flat"] for t in R.tris] + [False])[R.tri] & drawn
        assert ((vdr > 0.97) & flat).sum() >= 100 and ((vdr > 0.97) & ~flat & drawn).sum() >= 20, "highlights on flat and curved triangles"
        assert ((vdr > 0.9) & (vdr <= 0.97)).sum() >= 100, "the highlights' fall-off below the fast stage's cut-off"
        assert (F.lo[drawn] >= 254.5).sum() >= 100, "saturated channels"
    elif family == "light_gates":
        I = R.frag.intensity[R.inst > 0]
        assert (I == 0).sum() >= 100, "lit-away faces (intensity 0)"
        assert ((I > 0) & (I <= ref.SPEC_GATE)).sum() >= 100, "intensity in (0, 0.001]: the highlight gated off"
        assert ((I > ref.SPEC_GATE) & (I <= 3 * ref.SPEC_GATE)).sum() >= 100, "intensity just above 0.001: the highlight computed"
    elif family == "scaled_normals":
        drawn = R.inst > 0
        naive = render_naive(R)
        off = (np.abs(naive.frag.byte.astype(np.int16) - R.frag.byte.astype(np.int16)).max(-1) > 2) & drawn
        assert off.sum() >= 200 and off.sum() >= 0.25 * drawn.sum(), "normals by the model matrix instead of the normal matrix shade " \
            "%d of %d pixels within 2 LSB" % (int(drawn.sum() - off.sum()), int(drawn.sum()))
        assert sum(1 for t in front if t["mirrored"]) >= 4, "front faces of mirrored instances drawn"
    elif family == "near_plane":
        cut = [t for t in front if t["clip"] in ("near", "both")]
        assert sum(1 for t in cut if t["flat"]) >= 2 and sum(1 for t in cut if not t["flat"]) >= 4, \
            "flat and curved triangles cut by the near plane cover samples"
    elif family == "palette":
        lit = (R.inst > 0) & (np.nan_to_num(R.frag.intensity) > 0.3)
        assert all((lit & (R.color == k)).sum() >= 20 for k in range(22)), "every palette colour on lit faces"


def render_naive(R):
    """the scene of R drawn once more with normals transformed by the model-view 3 x 3 instead of its inverse transpose"""
    return ref.render(*R.scene, R.W, R.H, naive_normals=True)
