// Ray sensors (ray_kernel.h): one CTA per env casts the A * R rays of its agents against the env's instance list.
//
// The CTA walks the list in chunks of kChunk entries.  Each entry is inverted once (Magnum's adjugate / determinant, dm::inverted4) into
// shared memory, and every lane then tests its rays against the chunk in draw order: boxes by the slab test against [-1, 1]^3, the other
// meshes triangle by triangle (Moller-Trumbore, front faces only, widened bounds as a fallback at the edges) behind a conservative slab
// test of the mesh's bounds.  A model of negative determinant mirrors: its far faces are the drawn ones.  A lane holds up
// to kRaysPerThread rays, so every entry is inverted once per env whatever R is.  All lanes read the same entry and the same triangle at
// the same time: the shared-memory and constant-memory loads are broadcasts.
//
// The arithmetic is DESIGN.md section 3's definition, in the order written there (the build has -fmad=false); the CPU restatement is
// tests/oracle_seg/orc_rays.cpp.  A module of its own, like state_copy.cu: NVVM optimises per module, so the engine's tuned kernels do not
// see it.
#include "ray_kernel.h"

#include "../../include/megaverse_b200.h"
#include "dev_math.cuh"
#include "mesh_tables.inc"

namespace mvray {
namespace {
using namespace dm;

constexpr int kMaxThreads = 512;
constexpr int kRaysPerThread = (MV_MAX_AGENTS * MV_MAX_RAYS + kMaxThreads - 1) / kMaxThreads;
constexpr int kChunk = 128;
constexpr int kMirrored = 1 << 8;  // Chunk::mesh flag: the model's determinant is negative
// the prefilter box of a non-box mesh: its bounds ([-1, 1]^3, y in [-2, 2] for the capsule) grown by this much on every side in object
// units -- far more than the rounding of a hit point, so the prefilter never rejects a triangle the definition hits
constexpr float kBoundMargin = 1.0f / 64.0f;
// the widening of a triangle's barycentric bounds, in units of its det per object unit of |o - p0|_1 (plus one): about the rounding of
// u and w, which grows with the distance of the origin
constexpr float kEdgeTol = 1.0f / 262144.0f;

struct Chunk {
    float m[12][kChunk];  // rows 0..2 of the inverse model matrix, m[col * 3 + row]
    int mesh[kChunk];     // mesh type | kMirrored for a model of negative determinant; -1: an entry whose inverse is not finite, never hit
    int tag[kChunk];
};

// Magnum's determinant of a 4 x 4 matrix: the first-row cofactor expansion inverted4 divides by
__device__ __forceinline__ float det4(const M4 &m) {
    float d = 0.0f;
#pragma unroll
    for (int col = 0; col < 4; ++col) d += m.c[col * 4] * cofactor4(m, col, 0);
    return d;
}

__device__ __forceinline__ V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// rows 0..2 of m * (p, 1) and m * (p, 0), accumulated from 0 in column order (Magnum's transformPoint, as in dev_math.cuh)
__device__ __forceinline__ V3 xfPoint(const float m[12], V3 p) {
    V3 o;
    { float a = 0.0f; a += m[0] * p.x; a += m[3] * p.y; a += m[6] * p.z; a += m[9] * 1.0f; o.x = a; }
    { float a = 0.0f; a += m[1] * p.x; a += m[4] * p.y; a += m[7] * p.z; a += m[10] * 1.0f; o.y = a; }
    { float a = 0.0f; a += m[2] * p.x; a += m[5] * p.y; a += m[8] * p.z; a += m[11] * 1.0f; o.z = a; }
    return o;
}
__device__ __forceinline__ V3 xfVector(const float m[12], V3 v) {
    V3 o;
    { float a = 0.0f; a += m[0] * v.x; a += m[3] * v.y; a += m[6] * v.z; o.x = a; }
    { float a = 0.0f; a += m[1] * v.x; a += m[4] * v.y; a += m[7] * v.z; o.y = a; }
    { float a = 0.0f; a += m[2] * v.x; a += m[5] * v.y; a += m[8] * v.z; o.z = a; }
    return o;
}

// the slab test of o + t v against [-h, h] per axis: (t_in, t_out), axes x, y, z in turn
__device__ __forceinline__ void slab(V3 o, V3 v, V3 h, float &tin, float &tout) {
    tin = -INFINITY; tout = INFINITY;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float oi = comp(o, i), vi = comp(v, i), hi = comp(h, i);
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

// Moller-Trumbore against the triangle (p0, p1, p2) of object space, counted only when it faces the ray: s * det > 0, counter-clockwise
// seen from the ray's origin (s = +1), or clockwise for a mirrored model (s = -1), whose winding the world sees turned round -- the
// rasteriser's front face either way.  Barycentrics stay unnormalised: u, w in [0, det], u + w <= det.  0: no hit; 1: a hit within
// those bounds; 2: a hit only within the bounds widened by tol = det * kEdgeTol * (1 + |o - p0|_1), about the rounding of u and w, which
// meshHit takes only when no triangle of the mesh is hit within the exact bounds.  The signs are exact: with s = +1 every value is bit
// for bit the unsigned test's.
__device__ __forceinline__ int triHit(V3 o, V3 v, V3 p0, V3 p1, V3 p2, float s, float &t) {
    const V3 e1 = p1 - p0, e2 = p2 - p0;
    const V3 pv = cross(v, e2);
    const float det = s * dot(e1, pv);
    if (!(det > 0.0f)) return 0;
    const V3 tv = o - p0;
    float a = 1.0f;
    a += fabsf(tv.x); a += fabsf(tv.y); a += fabsf(tv.z);
    const float tol = det * (a * kEdgeTol);
    const float u = s * dot(tv, pv);
    if (u < -tol || u > det + tol) return 0;
    const V3 qv = cross(tv, e1);
    const float w = s * dot(v, qv);
    if (w < -tol || u + w > det + tol) return 0;
    t = s * dot(e2, qv) / det;
    return u < 0.0f || u > det || w < 0.0f || u + w > det ? 2 : 1;
}

template <int M> struct Mesh;
template <> struct Mesh<1> { static constexpr int tris = MV_CAPSULE_TRIS; __device__ static const float *v(int i) { return c_capsuleVerts[i]; } __device__ static int idx(int i) { return c_capsuleIdx[i]; } };
template <> struct Mesh<2> { static constexpr int tris = MV_SPHERE_TRIS; __device__ static const float *v(int i) { return c_sphereVerts[i]; } __device__ static int idx(int i) { return c_sphereIdx[i]; } };
template <> struct Mesh<3> { static constexpr int tris = MV_CONE_TRIS; __device__ static const float *v(int i) { return c_coneVerts[i]; } __device__ static int idx(int i) { return c_coneIdx[i]; } };
template <> struct Mesh<4> { static constexpr int tris = MV_CYLINDER_TRIS; __device__ static const float *v(int i) { return c_cylinderVerts[i]; } __device__ static int idx(int i) { return c_cylinderIdx[i]; } };

// every front-facing triangle of mesh M in index order: the nearest t in (0, best] wins, a later one on a tie.  Hits within the widened
// bounds only count when no triangle is hit within the exact ones: they close the cracks between faces and move no exact hit.
template <int M> __device__ __forceinline__ bool meshHit(V3 o, V3 v, float s, float &best) {
    bool exact = false, widened = false, nearer = false;
    float wide = best;
    for (int k = 0; k < Mesh<M>::tris; ++k) {
        const float *a = Mesh<M>::v(Mesh<M>::idx(3 * k)), *b = Mesh<M>::v(Mesh<M>::idx(3 * k + 1)), *c = Mesh<M>::v(Mesh<M>::idx(3 * k + 2));
        float t;
        const int h = triHit(o, v, v3(a[0], a[1], a[2]), v3(b[0], b[1], b[2]), v3(c[0], c[1], c[2]), s, t);
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
    return nearer;
}

__global__ void __launch_bounds__(kMaxThreads) rayKernel(const RayParams P) {
    __shared__ Chunk S;
    const int e = blockIdx.x;
    if (P.envMask && !P.envMask[e]) return;
    const int nRays = P.A * P.R, tid = threadIdx.x;
    const int nInst = __ldcg(P.instCounts + e * 8 + 1);
    const MvInstance *inst = P.instances + size_t(e) * size_t(P.instStride);

    // this lane's rays q = tid + k * blockDim.x: agent q / R, direction q % R, taken to world space through the inverse view matrix
    V3 ow[kRaysPerThread], dw[kRaysPerThread];
    float best[kRaysPerThread];
    int bestTag[kRaysPerThread], own[kRaysPerThread];
#pragma unroll
    for (int k = 0; k < kRaysPerThread; ++k) {
        const int q = tid + k * int(blockDim.x);
        best[k] = P.maxDist; bestTag[k] = -1; own[k] = -1;
        ow[k] = v3(0.0f, 0.0f, 0.0f); dw[k] = v3(0.0f, 0.0f, 0.0f);
        if (q >= nRays) continue;
        const int agent = q / P.R, r = q % P.R;
        M4 view;
#pragma unroll
        for (int i = 0; i < 16; ++i) view.c[i] = __ldcg(P.views + (size_t(e) * P.A + agent) * 16 + i);
        const M4 cam = inverted4(view);
        float c12[12];
#pragma unroll
        for (int col = 0; col < 4; ++col)
#pragma unroll
            for (int row = 0; row < 3; ++row) c12[col * 3 + row] = cam.c[col * 4 + row];
        ow[k] = xfPoint(c12, v3(0.0f, 0.0f, 0.0f));
        dw[k] = xfVector(c12, v3(P.dirs[3 * r], P.dirs[3 * r + 1], P.dirs[3 * r + 2]));
        own[k] = MV_SEG_AGENT << 8 | agent;
    }

    for (int base = 0; base < nInst; base += kChunk) {
        const int cnt = min(kChunk, nInst - base);
        __syncthreads();  // the previous chunk is read
        for (int i = tid; i < cnt; i += blockDim.x) {
            const MvInstance &d = inst[base + i];
            M4 model;
#pragma unroll
            for (int j = 0; j < 16; ++j) model.c[j] = __ldcg(&d.model[j]);
            const M4 mi = inverted4(model);
            bool finite = true;
#pragma unroll
            for (int col = 0; col < 4; ++col)
#pragma unroll
                for (int row = 0; row < 3; ++row) {
                    const float x = mi.c[col * 4 + row];
                    finite = finite && isfinite(x);
                    S.m[col * 3 + row][i] = x;
                }
            S.mesh[i] = finite ? (__ldcg(&d.mesh) | (det4(model) < 0.0f ? kMirrored : 0)) : -1;
            S.tag[i] = __ldcg(&d.pad[0]);
        }
        __syncthreads();
        for (int i = 0; i < cnt; ++i) {
            const int word = S.mesh[i], tag = S.tag[i];
            if (word < 0) continue;
            const int mesh = word & ~kMirrored;
            const bool mirrored = (word & kMirrored) != 0;
            float m[12];
#pragma unroll
            for (int j = 0; j < 12; ++j) m[j] = S.m[j][i];
#pragma unroll
            for (int k = 0; k < kRaysPerThread; ++k) {
                if (own[k] < 0 || tag == own[k]) continue;
                const V3 o = xfPoint(m, ow[k]), v = xfVector(m, dw[k]);
                if (mesh == 0) {
                    // a mirrored box shows its far faces: the exit, from outside and from inside alike
                    float tin, tout;
                    slab(o, v, v3(1.0f, 1.0f, 1.0f), tin, tout);
                    const float th = mirrored ? tout : tin;
                    if (th > 0.0f && tin <= tout && th <= best[k]) { best[k] = th; bestTag[k] = tag; }
                    continue;
                }
                float tin, tout;
                const float ys = mesh == 1 ? 2.0f : 1.0f;
                slab(o, v, v3(1.0f + kBoundMargin, ys + kBoundMargin, 1.0f + kBoundMargin), tin, tout);
                if (!(tin <= tout && tout > 0.0f)) continue;
                bool hit;
                const float s = mirrored ? -1.0f : 1.0f;
                if (mesh == 1) hit = meshHit<1>(o, v, s, best[k]);
                else if (mesh == 2) hit = meshHit<2>(o, v, s, best[k]);
                else if (mesh == 3) hit = meshHit<3>(o, v, s, best[k]);
                else hit = meshHit<4>(o, v, s, best[k]);
                if (hit) bestTag[k] = tag;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < kRaysPerThread; ++k) {
        const int q = tid + k * int(blockDim.x);
        if (q >= nRays) continue;
        const size_t o = size_t(e) * size_t(nRays) + size_t(q);  // = (e * A + agent) * R + r
        P.dist[o] = bestTag[k] >= 0 ? best[k] : 0.0f;
        P.tag[o] = uint16_t(bestTag[k] >= 0 ? bestTag[k] : 0);
    }
}

}  // namespace

cudaError_t castRays(const RayParams &p, cudaStream_t stream) {
    const int nRays = p.A * p.R;
    if (p.E < 1 || nRays < 1 || p.R > MV_MAX_RAYS || p.A > MV_MAX_AGENTS) return cudaErrorInvalidValue;
    const int threads = min(kMaxThreads, (nRays + 31) / 32 * 32);
    rayKernel<<<p.E, threads, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace mvray
