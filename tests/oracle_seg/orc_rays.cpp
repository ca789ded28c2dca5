// Ray sensors on the ORACLE (test infrastructure, never linked or imported by the product): the engine's ray definition (DESIGN.md
// section 3, "Ray sensors"), operation by operation in the same order, over the oracle's own tagged scene of one env (orc_seg.cpp's
// sceneTags over Env::instances(), seen from the oracle's view(env, agent)) or over a hand-built instance list.  Built like orc_seg.cpp
// (tests/orc_rays.py, the compiler and flags of oracle/Makefile: no contraction), which it includes unchanged.
#include "orc_seg.cpp"

namespace {

constexpr float kBoundMargin = 1.0f / 64.0f;  // the prefilter's margin, as in csrc/ray_kernel.cu (it changes no result)
constexpr float kEdgeTol = 1.0f / 262144.0f;   // the widening of the barycentric bounds per object unit of |o - p0|, as in csrc/ray_kernel.cu

Vec3 cross3(Vec3 a, Vec3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// rows 0..2 of m * (p, 1) and of m * (v, 0), accumulated from 0 in column order
Vec3 xfPoint(const Mat4 &m, Vec3 p) {
    Vec3 o;
    for (int row = 0; row < 3; ++row) {
        float a = 0.0f;
        a += m.c[0][row] * p.x; a += m.c[1][row] * p.y; a += m.c[2][row] * p.z; a += m.c[3][row] * 1.0f;
        o[row] = a;
    }
    return o;
}
Vec3 xfVector(const Mat4 &m, Vec3 v) {
    Vec3 o;
    for (int row = 0; row < 3; ++row) {
        float a = 0.0f;
        a += m.c[0][row] * v.x; a += m.c[1][row] * v.y; a += m.c[2][row] * v.z;
        o[row] = a;
    }
    return o;
}

void slab(Vec3 o, Vec3 v, Vec3 h, float &tin, float &tout) {
    tin = -INFINITY; tout = INFINITY;
    for (int i = 0; i < 3; ++i) {
        const float oi = o[i], vi = v[i], hi = h[i];
        if (vi == 0.0f) {
            if (oi < -hi || oi > hi) { tin = INFINITY; tout = -INFINITY; }
            continue;
        }
        const float inv = 1.0f / vi;
        const float t0 = (-hi - oi) * inv, t1 = (hi - oi) * inv;
        const float lo = t0 < t1 ? t0 : t1, up = t0 < t1 ? t1 : t0;
        tin = lo > tin ? lo : tin;
        tout = up < tout ? up : tout;
    }
}

// s = -1 for a mirrored model: the faces counted are those clockwise seen from the origin.  0: no hit; 1: a hit within the exact bounds;
// 2: within the bounds widened by tol only (a fallback, see castFan)
int triHit(Vec3 o, Vec3 v, Vec3 p0, Vec3 p1, Vec3 p2, float s, float &t) {
    const Vec3 e1 = p1 - p0, e2 = p2 - p0;
    const Vec3 pv = cross3(v, e2);
    const float det = s * dot(e1, pv);
    if (!(det > 0.0f)) return 0;
    const Vec3 tv = o - p0;
    float a = 1.0f;
    a += std::fabs(tv.x); a += std::fabs(tv.y); a += std::fabs(tv.z);
    const float tol = det * (a * kEdgeTol);
    const float u = s * dot(tv, pv);
    if (u < -tol || u > det + tol) return 0;
    const Vec3 qv = cross3(tv, e1);
    const float w = s * dot(v, qv);
    if (w < -tol || u + w > det + tol) return 0;
    t = s * dot(e2, qv) / det;
    return u < 0.0f || u > det || w < 0.0f || u + w > det ? 2 : 1;
}

Vec3 vertex(const MeshRef &m, int i) { return {bitsToFloat(m.vtx[i][0]), bitsToFloat(m.vtx[i][1]), bitsToFloat(m.vtx[i][2])}; }

// the R rays of `agent` (-1: no drawable is its own) seen through `view` against the tagged instance list
void castFan(const Mat4 &view, const std::vector<Instance> &inst, const std::vector<int> &tags, int agent, const float *dirs, int R, float maxDist,
             float *dist, uint16_t *tag) {
    const Mat4 cam = inverted(view);
    const int own = agent < 0 ? -1 : (SEG_AGENT << 8 | agent);
    std::vector<Mat4> inv(inst.size());
    std::vector<bool> finite(inst.size()), mirrored(inst.size());
    for (size_t i = 0; i < inst.size(); ++i) {
        inv[i] = inverted(inst[i].model);
        mirrored[i] = det4(inst[i].model) < 0.0f;
        bool f = true;
        for (int col = 0; col < 4; ++col)
            for (int row = 0; row < 3; ++row) f = f && std::isfinite(inv[i].c[col][row]);
        finite[i] = f;
    }
    for (int r = 0; r < R; ++r) {
        const Vec3 ow = xfPoint(cam, {0.0f, 0.0f, 0.0f});
        const Vec3 dw = xfVector(cam, {dirs[3 * r], dirs[3 * r + 1], dirs[3 * r + 2]});
        float best = maxDist;
        int bestTag = -1;
        for (size_t i = 0; i < inst.size(); ++i) {
            if (!finite[i] || tags[i] == own) continue;
            const Vec3 o = xfPoint(inv[i], ow), v = xfVector(inv[i], dw);
            float tin, tout;
            if (inst[i].mesh == MESH_BOX) {
                slab(o, v, {1.0f, 1.0f, 1.0f}, tin, tout);
                const float th = mirrored[i] ? tout : tin;  // a mirrored box shows its far faces
                if (th > 0.0f && tin <= tout && th <= best) { best = th; bestTag = tags[i]; }
                continue;
            }
            const float ys = inst[i].mesh == MESH_CAPSULE ? 2.0f : 1.0f;
            slab(o, v, {1.0f + kBoundMargin, ys + kBoundMargin, 1.0f + kBoundMargin}, tin, tout);
            if (!(tin <= tout && tout > 0.0f)) continue;
            const MeshRef m = meshRef(inst[i].mesh);
            const float s = mirrored[i] ? -1.0f : 1.0f;
            // hits within the exact bounds count as they are; a hit within the widened bounds only counts when no triangle of the
            // instance is hit within the exact ones, so the widening closes the cracks between its faces and moves no exact hit
            float wide = best;
            bool exact = false, widened = false, nearer = false;
            for (int k = 0; k + 2 < m.ni; k += 3) {
                float t;
                const int h = triHit(o, v, vertex(m, m.idx[k]), vertex(m, m.idx[k + 1]), vertex(m, m.idx[k + 2]), s, t);
                if (!h || !(t > 0.0f)) continue;
                if (h == 1) {
                    exact = true;
                    if (t <= best) { best = t; nearer = true; }
                } else if (t <= wide) {
                    wide = t;
                    widened = true;
                }
            }
            if (!exact && widened) { best = wide; nearer = true; }
            if (nearer) bestTag = tags[i];
        }
        dist[r] = bestTag >= 0 ? best : 0.0f;
        tag[r] = uint16_t(bestTag >= 0 ? bestTag : 0);
    }
}

}  // namespace

extern "C" {
// dist float[R], tag uint16[R]: agent `agent`'s rays in env `env` of the oracle's current scenes, from view16 (column-major) or, when it is
// NULL, from the oracle's own view(env, agent).  0 on success, -1 for an env or agent out of range or when the tags cannot be assigned.
int orc_rays_env(void *p, int env, int agent, const float *view16, const float *dirs, int R, float maxDist, float *dist, uint16_t *tag) {
    auto *v = static_cast<OrcVec *>(p);
    if (env < 0 || env >= v->numEnvs || agent < 0 || agent >= v->numAgents) return -1;
    try {
        const Env &e = *v->envs[size_t(env)];
        const auto inst = e.instances();
        const auto tags = sceneTags(e);
        if (tags.size() != inst.size()) return -1;
        Mat4 view = e.viewMatrix(agent);
        if (view16) std::memcpy(&view.c[0][0], view16, 64);
        castFan(view, inst, tags, agent, dirs, R, maxDist, dist, tag);
    } catch (const std::exception &) {
        return -1;
    }
    return 0;
}
// the same over a hand-built scene: n instances of 18 floats (mesh, colour, column-major model: orc_render_instances' layout) with their
// tags; agent -1 ignores no drawable
void orc_rays_scene(const float *view16, const float *inst18, const int32_t *tags, int n, int agent, const float *dirs, int R, float maxDist,
                    float *dist, uint16_t *tag) {
    Mat4 view;
    std::memcpy(&view.c[0][0], view16, 64);
    std::vector<Instance> inst(static_cast<size_t>(n));
    for (int i = 0; i < n; ++i) {
        inst[size_t(i)].mesh = int(inst18[i * 18]); inst[size_t(i)].color = int(inst18[i * 18 + 1]);
        std::memcpy(&inst[size_t(i)].model.c[0][0], inst18 + i * 18 + 2, 64);
    }
    castFan(view, inst, std::vector<int>(tags, tags + n), agent, dirs, R, maxDist, dist, tag);
}
}
