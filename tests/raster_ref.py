"""An INDEPENDENT restatement of the fixed-function rasterisation rules, for any frame size (test infrastructure, CPU only).

The reference draws with Vulkan (V4R: vulkan_state.cpp:588-606 -- back-face culling with counter-clockwise fronts, depth test
LESS_OR_EQUAL on a D32 attachment, one sample per pixel).  The rules restated here are the Vulkan specification's, not reference code:
view-volume clipping 0 <= z_c <= w_c, the viewport transform, fixed-point vertex positions (8 sub-pixel bits), one sample at the pixel
centre, the top-left rule for samples exactly on an edge, depth interpolated linearly in window space, perspective-correct interpolation
of the varyings (here: clip-space w, which V4R writes out as its depth image).

They are implemented in a different form and in different arithmetic from the oracle (oracle/orc_raster.hpp) and the CUDA kernel:

  * window coordinates: the float32 snap value taken as an UNBOUNDED integer -- no int32 conversion, no saturation, no wrap: the answer
    of a rasteriser with a guard band wide enough for every vertex the near plane lets through;
  * coverage: exact integers, a sample on an edge is decided by displacing it infinitesimally to the right and, second order, down
    (lexicographic sign of (E, dE/dx, dE/dy)) -- no top-left classification of edges, no bias constants;
  * depth and w: float64 barycentrics from the exact integer edge values;
  * hidden-surface removal: per pixel over all covering triangles, nearest depth, the later draw on ties;
  * clipping: Sutherland-Hodgman in float64 on the clip coordinates.

Only the vertex stage is shared knowledge (float32 arithmetic in the order of uber.vert / Magnum, pinned elsewhere against the real
shader text and the real Magnum): it is recomputed here in numpy float32 so that every side snaps the same window coordinates.

render() also returns a record of every source triangle -- which planes clipped it, whether it was culled by its winding, whether its
instance mirrors, the kernel-style edge bound, whether its pixel box meets some 32 x 4 tile in at most four pixels -- so that a
constructed scene can prove which branch of a rasteriser it reached without any counter inside the rasteriser.
"""
import numpy as np

import orc

F32 = np.float32
SUB = 256            # 8 sub-pixel bits
TILE_W, TILE_H = 32, 4
SMALL_AREA = 4       # pixels of a tile at or below which a triangle takes a rasteriser's one-lane path
EDGE_INT32 = 1 << 30  # kernel-style edge bound below which the edge functions fit int32 over the viewport


def projection(W, H):
    """p00, p11, p22, p32 of the reference's perspective (v4r.cpp:35-45): 100 degrees, aspect W / H, near 0.01, far 120, y flipped"""
    aspect = F32(W) / F32(H)
    half_tan = F32(np.tan(np.float64(F32(100.0) * F32(0.01745329251994329576923690768489)) / 2.0))  # correctly rounded tan, as the oracle's crtan
    near, far = F32(0.01), F32(120.0)
    return F32(1.0) / half_tan, -aspect / half_tan, far / (near - far), far * near / (near - far)


_MESHES = {}


def _mesh_tables(kind):
    if kind not in _MESHES:
        vtx, idx = orc.mesh(kind)
        v6 = vtx.view(np.float32).reshape(-1, 6)
        _MESHES[kind] = (v6[:, :3].copy(), idx.reshape(-1, 3).astype(np.int64), v6[:, 3:].astype(np.float64))
    return _MESHES[kind]


def mesh(kind):
    """(vertex positions float32 [n][3], triangle indices int64 [t][3]) of mesh type kind (0 box .. 4 cylinder)"""
    return _mesh_tables(kind)[:2]


def normals(kind):
    """vertex normals float64 [n][3] of mesh type kind (the mesh tables' float32 values)"""
    return _mesh_tables(kind)[2]


def model_view(view16, model16):
    """view * model in float32, the accumulation order of Magnum's Matrix4 product; [col][row]"""
    v = np.asarray(view16, dtype=F32).reshape(4, 4)
    m = np.asarray(model16, dtype=F32).reshape(4, 4)
    mv = np.zeros((4, 4), dtype=F32)
    for col in range(4):
        for row in range(4):
            acc = F32(0.0)
            for pos in range(4):
                acc = F32(acc + F32(v[pos][row] * m[col][pos]))
            mv[col][row] = acc
    return mv


def vertex_stage(view16, model16, verts, W, H):
    """clip-space positions, float32, in the operation order of the vertex stage (uber.vert:53-110 on column-major matrices)"""
    mv = model_view(view16, model16)
    p00, p11, p22, p32 = projection(W, H)
    p = np.asarray(verts, dtype=F32)
    cam = []
    for row in range(3):
        acc = np.zeros(len(p), dtype=F32)
        acc = acc + mv[0][row] * p[:, 0]
        acc = acc + mv[1][row] * p[:, 1]
        acc = acc + mv[2][row] * p[:, 2]
        acc = acc + mv[3][row] * F32(1.0)
        cam.append(acc)
    return np.stack([cam[0] * p00, cam[1] * p11, cam[2] * p22 + p32, -cam[2]], axis=1).astype(F32)


def snap(clip, W, H):
    """viewport transform + fixed point in float32 (as every side computes it), the snap value then taken as an unbounded integer;
    returns (x, y, z_ndc, 1/w)"""
    c = np.asarray(clip, dtype=F32)
    r = F32(1.0) / c[3]
    hw, hh = F32(W) * F32(0.5), F32(H) * F32(0.5)
    x = F32(F32(F32(c[0] * r) * hw) + hw)
    y = F32(F32(F32(c[1] * r) * hh) + hh)
    fx, fy = F32(F32(x * F32(SUB)) + F32(0.5)), F32(F32(y * F32(SUB)) + F32(0.5))
    assert np.isfinite(fx) and np.isfinite(fy), "a vertex projected to infinity"
    return int(np.floor(np.float64(fx))), int(np.floor(np.float64(fy))), np.float64(F32(c[2] * r)), np.float64(r)


def clip_polygon(poly):
    """Sutherland-Hodgman against 0 <= z <= w in float64 (Vulkan 'primitive clipping', depth range zero-to-one)"""
    for plane in (0, 1):
        dist = (lambda c: c[2]) if plane == 0 else (lambda c: c[3] - c[2])
        out = []
        for i in range(len(poly)):
            a, b = poly[i], poly[(i + 1) % len(poly)]
            da, db = dist(a), dist(b)
            if da >= 0:
                out.append(a)
            if (da >= 0) != (db >= 0):
                t = da / (da - db)
                out.append(a + t * (b - a))
        poly = out
        if len(poly) < 3:
            return []
    return poly


def _edge_values(dEdx, dEdy, K, sx, sy):
    """E = dEdx * sx + dEdy * sy + K at the samples, exactly: (sign-exact integer array or None, float64 array).  dEdx, dEdy and K are
    Python integers of any size; sx, sy int64 sample positions (< 2^21)."""
    if abs(dEdx) < (1 << 40) and abs(dEdy) < (1 << 40):
        P = np.int64(dEdx) * sx + np.int64(dEdy) * sy                 # |P| < 2^62
        if abs(K) >= (1 << 62):                                       # |P| < |K|: E has the sign of K at every sample
            return np.full(sx.shape, 1 if K > 0 else -1, dtype=np.int64), P.astype(np.float64) + float(K)
        E = P + np.int64(K)
        return E, E.astype(np.float64)
    E = dEdx * sx.astype(object) + dEdy * sy.astype(object) + K        # Python integers: exact at any size
    sign = np.array([(e > 0) - (e < 0) for e in E.ravel()], dtype=np.int64).reshape(E.shape)
    return sign, np.array([float(e) for e in E.ravel()]).reshape(E.shape)


def _min_tile_part(lo, hi, size):
    """shortest part of the inclusive range [lo, hi] cut at multiples of size"""
    first = min(hi, (lo // size) * size + size - 1) - lo + 1
    last = hi - max(lo, (hi // size) * size) + 1
    return min(first, last)


class Render:
    """w: float64 [H][W] (view-space w of the visible fragment, 0 = empty); inst: int32 [H][W] (index + 1 of the winning instance, 0 =
    empty); z: float64 [H][W] window depth; tris: one dict per source triangle; pieces: one dict per drawn (front-facing, on-screen)
    screen triangle; ties: samples that lay exactly on an edge of a front-facing triangle.
    The varyings of the visible fragment, interpolated with perspective correction: P, N float64 [H][W][3] (camera-space position and
    unnormalised normal); color: int32 [H][W] palette index (-1 = empty).  frag runs the fragment stage on them."""

    def __init__(self, W, H):
        self.W, self.H = W, H
        self.z = np.full((H, W), np.inf)
        self.w = np.zeros((H, W))
        self.inst = np.zeros((H, W), dtype=np.int32)
        self.P = np.zeros((H, W, 3))
        self.N = np.zeros((H, W, 3))
        self.color = np.full((H, W), -1, dtype=np.int32)
        self.tri = np.full((H, W), -1, dtype=np.int32)  # index into tris of the visible fragment's source triangle
        self.tris, self.pieces, self.ties = [], [], 0
        self.scene = None
        self._frag = None

    @property
    def frag(self):
        """the float64 fragment stage of every pixel (Fragments), computed once"""
        if self._frag is None:
            self._frag = shade64(self.P, self.N, self.color)
        return self._frag

    @property
    def clipped(self):
        return any(t["clip"] != "none" for t in self.tris)

    def reached(self, key, value=True):
        return sum(1 for t in self.tris if t.get(key) == value)


def render(view16, instances, W, H, naive_normals=False):
    """draw the instances (rows of 18 floats: mesh, colour, 16 model floats column-major, in draw order) by the specification's rules.
    naive_normals: transform the normals by the model-view 3 x 3 itself instead of its inverse transpose (a deliberately wrong vertex
    stage, for proving that a scene tells the two apart)"""
    R = Render(W, H)
    R.scene = (view16, instances)
    for ii, row in enumerate(np.asarray(instances, dtype=F32).reshape(-1, 18)):
        verts, tris = mesh(int(row[0]))
        mv = model_view(view16, row[2:18])
        mirrored = bool(np.linalg.det(mv[:3, :3].astype(np.float64)) <= 0)
        clip = vertex_stage(view16, row[2:18], verts, W, H)
        # varyings in float64 from the float32 model-view matrix: camera-space position and normal (inverse transpose, by numpy)
        M = mv.T.astype(np.float64)  # [row][col]
        nm = M[:3, :3] if naive_normals else np.linalg.inv(M[:3, :3]).T
        cam64 = verts.astype(np.float64) @ M[:3, :3].T + M[:3, 3]
        vary = np.concatenate([clip.astype(np.float64), cam64, normals(int(row[0])) @ nm.T], axis=1)  # [n][10]: clip, P, N
        p00, p11, _, _ = projection(W, H)
        cam = np.stack([clip[:, 0] / np.float64(p00), clip[:, 1] / np.float64(p11), -clip[:, 3].astype(np.float64)], axis=1)
        for ti, tri in enumerate(tris):
            c = clip[tri]
            near_out, far_out = c[:, 2] < 0, (c[:, 3] - c[:, 2]) < 0
            # sine of the angle between the triangle's plane and the direction to the eye (view space, float64)
            a, b, d = cam[tri[0]], cam[tri[1]], cam[tri[2]]
            n = np.cross(b - a, d - a)
            den = np.linalg.norm(n) * np.linalg.norm(a)
            rec = {"inst": ii, "tri": ti, "mirrored": mirrored, "behind_near": bool(near_out.all()), "beyond_far": bool(far_out.all()),
                   "clip": {(False, False): "none", (True, False): "near", (False, True): "far", (True, True): "both"}[(bool(near_out.any()), bool(far_out.any()))],
                   "culled": False, "front": False, "small": False, "bound": 0, "max_coord": 0, "max_delta": 0, "pieces": 0, "covered": 0,
                   "sin": float(abs(np.dot(n, a)) / den) if den > 0 else None, "min_extent": 1 << 62,
                   "flat": bool((normals(int(row[0]))[tri] == normals(int(row[0]))[tri[0]]).all())}
            R.tris.append(rec)
            v = vary[tri]
            if rec["clip"] != "none":
                poly = clip_polygon([v[k] for k in range(3)])  # the varyings ride along as extra components
                pieces = [(poly[0], poly[k], poly[k + 1]) for k in range(1, len(poly) - 1)]
                rec["poly"] = len(poly)
            else:
                pieces = [(v[0], v[1], v[2])]
            rec["pieces"] = len(pieces)
            for piece in pieces:
                sv = [snap(np.asarray(v[:4], dtype=F32), W, H) for v in piece]
                xs, ys = [s[0] for s in sv], [s[1] for s in sv]
                rec["max_coord"] = max(rec["max_coord"], max(abs(v) for v in xs + ys))
                rec["max_delta"] = max(rec["max_delta"], max(abs(xs[i] - xs[j]) for i in range(3) for j in range(3)),
                                       max(abs(ys[i] - ys[j]) for i in range(3) for j in range(3)))
                area2 = (xs[1] - xs[0]) * (ys[2] - ys[0]) - (ys[1] - ys[0]) * (xs[2] - xs[0])
                if area2 >= 0:
                    rec["culled"] = True  # clockwise on a y-down screen = back face (fronts are counter-clockwise in y-up NDC), or degenerate
                    continue
                rec["front"] = True
                rec["min_extent"] = min(rec["min_extent"], max(xs) - min(xs), max(ys) - min(ys))
                # the kernel-style bound of the edge functions over the viewport: |dy| W + |dx| H + |C| in sub-pixels
                bound = 0
                for a, b in ((1, 2), (2, 0), (0, 1)):
                    dx, dy = xs[b] - xs[a], ys[b] - ys[a]
                    bound = max(bound, abs(dy) * W * SUB + abs(dx) * H * SUB + abs(dx * ys[a] - dy * xs[a]))
                rec["bound"] = max(rec["bound"], bound)
                # pixel box: pixel p has its sample at p * 256 + 128
                px0, px1 = max(0, -((128 - min(xs)) // SUB)), min(W - 1, (max(xs) - 128) // SUB)
                py0, py1 = max(0, -((128 - min(ys)) // SUB)), min(H - 1, (max(ys) - 128) // SUB)
                if px0 > px1 or py0 > py1:
                    continue
                if _min_tile_part(px0, px1, TILE_W) * _min_tile_part(py0, py1, TILE_H) <= SMALL_AREA:
                    rec["small"] = True
                gy, gx = np.mgrid[py0:py1 + 1, px0:px1 + 1]
                sx, sy = gx.astype(np.int64) * SUB + 128, gy.astype(np.int64) * SUB + 128
                inside = np.ones(gx.shape, dtype=bool)
                lam = []
                for a, b in ((1, 2), (2, 0), (0, 1)):
                    # edge function oriented so that the interior is positive; a sample ON the edge counts iff an infinitesimal step
                    # right (then down) enters the interior: sign of (E, dE/dx, dE/dy) in lexicographic order
                    dEdx, dEdy = ys[b] - ys[a], -(xs[b] - xs[a])
                    E, Ef = _edge_values(dEdx, dEdy, -dEdx * xs[a] - dEdy * ys[a], sx, sy)
                    tie = dEdx > 0 or (dEdx == 0 and dEdy > 0)
                    inside &= (E > 0) | ((E == 0) & tie)
                    R.ties += int((E == 0).sum())
                    lam.append(Ef / float(-area2))
                if not inside.any():
                    continue
                zs, rws = [s[2] for s in sv], [s[3] for s in sv]
                z = lam[0] * zs[0] + lam[1] * zs[1] + lam[2] * zs[2]          # depth: linear in window space
                with np.errstate(divide="ignore"):
                    w = 1.0 / (lam[0] * rws[0] + lam[1] * rws[1] + lam[2] * rws[2])  # perspective-correct w
                bz = R.z[py0:py1 + 1, px0:px1 + 1]
                win = inside & (z <= 1.0) & (z <= bz)                          # LESS_OR_EQUAL: the later draw replaces an equal depth
                rec["covered"] += int(inside.sum())
                R.pieces.append({"inst": ii, "tri": ti, "x": xs, "y": ys})
                R.z[py0:py1 + 1, px0:px1 + 1] = np.where(win, z, bz)
                R.w[py0:py1 + 1, px0:px1 + 1] = np.where(win, w, R.w[py0:py1 + 1, px0:px1 + 1])
                R.inst[py0:py1 + 1, px0:px1 + 1] = np.where(win, ii + 1, R.inst[py0:py1 + 1, px0:px1 + 1])
                # perspective-correct varyings: weights lambda_i / w_i, w_i in float64 from the (clipped) vertex itself
                k = [lam[i] / piece[i][3] for i in range(3)]
                s = k[0] + k[1] + k[2]
                for dst, c0 in ((R.P, 4), (R.N, 7)):
                    val = sum((k[i] / s)[..., None] * piece[i][c0:c0 + 3] for i in range(3))
                    dst[py0:py1 + 1, px0:px1 + 1] = np.where(win[..., None], val, dst[py0:py1 + 1, px0:px1 + 1])
                R.color[py0:py1 + 1, px0:px1 + 1] = np.where(win, int(row[1]), R.color[py0:py1 + 1, px0:px1 + 1])
                R.tri[py0:py1 + 1, px0:px1 + 1] = np.where(win, len(R.tris) - 1, R.tri[py0:py1 + 1, px0:px1 + 1])
    return R


# ---------------------------------------------------------------------------------------------------- the fragment stage in float64
def _palette():
    from test_ref_golden import PALETTE

    return np.array([[(c >> 16) & 255, (c >> 8) & 255, c & 255] for c in PALETTE], dtype=np.float64) / 255.0


LIGHT = np.array([0.0, 4.0, 2.0])  # camera space (v4r_env_renderer.cpp:220)
SPEC_GATE = 0.001                  # the highlight is computed only where intensity > SPEC_GATE (uber.frag)
SHININESS = 300


class Fragments:
    """per pixel of a Render: lo float64 [H][W][3] (the colour in LSB, 255 * clamp(Lo, 0, 1)), byte uint8 [H][W][3] (UNORM8: floor(lo +
    0.5)), margin float64 [H][W][3] (distance of 255 * Lo from the nearest rounding boundary k + 1/2, k = 0 .. 254, in LSB; inf where
    nothing was drawn), intensity = max(N.L, 0), vdr = V.reflect(-L, N) (nan where the highlight is gated off or nothing was drawn), spec
    (the highlight term, 0 where gated off)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def shade64(P, N, color):
    """uber.frag:112-141 (the non-Blinn-Phong branch) restated in float64 for every pixel: P, N [H][W][3] camera-space position and
    unnormalised normal, color [H][W] palette index (-1: nothing drawn, black).  Light at LIGHT, colour 0.66, specular 1, shininess 300:
        Lo = 0.33 d + 0.73 * 0.66 d * max(N.L, 0) + (N.L > 0.001 ? clamp(max(V.R, 0)^300, 0, 1) : 0),   R = reflect(-L, N)"""
    drawn = color >= 0
    d = _palette()[np.where(drawn, color, 0)]
    with np.errstate(invalid="ignore", divide="ignore"):
        cd = -P
        nl = (LIGHT + cd) / np.linalg.norm(LIGHT + cd, axis=-1, keepdims=True)
        nn = N / np.linalg.norm(N, axis=-1, keepdims=True)
        ndl = (nn * nl).sum(-1)
        intensity = np.maximum(ndl, 0.0)
        refl = -nl + 2.0 * ndl[..., None] * nn
        vdr = (cd / np.linalg.norm(cd, axis=-1, keepdims=True) * refl).sum(-1)
    lit = drawn & (intensity > SPEC_GATE)
    vdr = np.where(lit, vdr, np.nan)
    spec = np.where(lit, np.clip(np.maximum(np.nan_to_num(vdr), 0.0) ** SHININESS, 0.0, 1.0), 0.0)
    Lo = 0.33 * d + (0.73 * 0.66) * d * np.where(drawn, intensity, 0.0)[..., None] + spec[..., None]
    x = np.where(drawn[..., None], 255.0 * Lo, 0.0)
    margin = np.where(drawn[..., None], np.abs(x - np.clip(np.floor(x) + 0.5, 0.5, 254.5)), np.inf)
    lo = np.clip(x, 0.0, 255.0)
    return Fragments(lo=lo, byte=np.floor(lo + 0.5).astype(np.uint8), margin=margin, intensity=np.where(drawn, intensity, np.nan), vdr=vdr,
                     spec=spec)


# The colour rule.  A rasteriser that computes the fragment stage in float32 (the oracle; the kernel's exact variant reproduces it byte
# for byte) writes, wherever it draws the same surface as the reference, bytes within 1 LSB of the float64 ones, and a byte may differ at
# all only where 255 Lo lies within M LSB of a rounding boundary (k + 1/2):
#   M = M0 + 255 * 300 * max(vdr, 0)^299 * EPS_VDR   [+ 255 * spec where vdr <= FAST_CUT, fast fragment stage only]
#   * M0 = 0.02 LSB: the ambient and diffuse terms move by 255 * 0.81 * (error of N.L); N.L carries float32 rounding of the vertex stage,
#     the normal matrix, the interpolation and two normalisations, a few ulp, below 1e-6 -- 2e-4 LSB; M0 leaves a hundredfold margin
#     (measured on every family against the oracle: at most 0.006 LSB, all of it in highlights);
#   * the highlight vdr^300 multiplies an error of vdr by 300 vdr^299: EPS_VDR = 2^-20 (16 ulp of 1.0 in float32; the fast stage's
#     rsqrt.approx is within 2 ulp) covers the dot products and normalisations vdr goes through -- up to 0.073 LSB at vdr = 1;
#   * the fast stage drops the highlight where vdr <= 0.97 (0.97^300 = 1.1e-4, at most 0.028 LSB): there the float64 value it is held to
#     is shifted by exactly the term dropped.
M0, EPS_VDR, FAST_CUT = 0.02, 2.0 ** -20, 0.97


def colour_rule(frag, rgb, same, fast=False):
    """rgb uint8 [H][W][3] against the float64 fragments where `same` (both sides drew the same surface) holds: (bytes that break the rule,
    bytes that differ, the largest margin among the differing bytes in LSB, the largest difference)"""
    vdr = np.maximum(np.nan_to_num(frag.vdr, nan=0.0), 0.0)
    M = M0 + 255.0 * SHININESS * vdr ** (SHININESS - 1) * EPS_VDR
    if fast:
        M = M + np.where(vdr <= FAST_CUT, 255.0 * frag.spec, 0.0)
    d = np.abs(rgb[..., :3].astype(np.int16) - frag.byte.astype(np.int16))
    d = np.where(same[..., None], d, 0)
    differ = d > 0
    broken = (d > 1) | (differ & (frag.margin >= M[..., None]))
    return int(broken.sum()), int(differ.sum()), float(frag.margin[differ].max(initial=0.0)), int(d.max(initial=0))
