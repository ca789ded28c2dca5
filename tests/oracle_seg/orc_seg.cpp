// Segmentation on the ORACLE (test infrastructure, never linked or imported by the product): for every view of an oracle vector env,
// the class and index of the scene object whose fragment wins each pixel, class << 8 | index (the engine's MV_SEG_*), 0 where nothing
// was drawn.  The tags come from the oracle's own scene objects (DrawEntry kinds and indices, its terrain slabs), never from the
// engine's instance-slot layout.  The raster part restates oracle/orc_raster.hpp's renderView with the per-pixel winner kept: the same
// vertex stage, clipAndSetup and coverage / LESS_OR_EQUAL loop; it also returns the depth it drew, which the tests compare bit for bit
// with renderView's own.
//
// The whole oracle API is compiled into this library so that OrcVec is the type oracle/liborc.so creates: the Python side passes the
// handle of an orc.Oracle here.  Both libraries are built by the same compiler with the same flags (tests/orc_seg.py, oracle/Makefile).
#include "../../oracle/orc_api.cpp"

namespace {

enum SegClass { SEG_STATIC = 1, SEG_TERRAIN = 2, SEG_OBJECT = 3, SEG_AGENT = 4, SEG_REWARD = 5 };

bool sameMatrix(const Mat4 &a, const Mat4 &b) { return std::memcmp(&a.c[0][0], &b.c[0][0], sizeof(float) * 16) == 0; }

// the tag of every entry of Env::instances(), in its order (mesh type major, insertion order minor)
std::vector<int> sceneTags(const Env &env) {
    // Terrain slabs are drawn as D_STATIC boxes: Env::addTerrain draws a slab that has width, in the order of env.terrainSlabs, with
    // this model matrix (layout_utils.cpp:53-68)
    std::vector<std::pair<int, Mat4>> slabs;
    for (const TerrainSlab &ts : env.terrainSlabs) {
        const BoundingBox &bb = ts.bb;
        const Vec3 scale = Vec3{float(bb.max.x - bb.min.x), 1.0f, float(bb.max.z - bb.min.z)} * 1.0f;
        if (!(scale.x > 0)) continue;
        const Vec3 pos{bb.min.x * 1.0f + scale.x / 2, bb.min.y * 1.0f, bb.min.z * 1.0f + scale.z / 2};
        Mat4 m = mul(mat4Scaling({0.5f, 0.025f, 0.5f}), mat4Identity());
        m = mul(mat4Scaling(scale), m);
        m = mul(mat4Translation({0.0f, 0.025f, 0.0f}), m);
        m = mul(mat4Translation(pos), m);
        slabs.push_back({ts.terrain, m});
    }
    size_t nextSlab = 0;
    std::vector<int> tags;
    for (const auto &[mesh, list] : env.drawables)
        for (const DrawEntry &d : list) {
            int tag = SEG_STATIC << 8;
            switch (d.kind) {
                case DrawEntry::D_STATIC:
                    if (mesh == MESH_BOX && nextSlab < slabs.size() && sameMatrix(d.model, slabs[nextSlab].second)) {
                        int bit = 0;  // the slab's TerrainType bit number
                        while (!((slabs[nextSlab].first >> bit) & 1)) ++bit;
                        tag = SEG_TERRAIN << 8 | bit;
                        ++nextSlab;
                    }
                    break;
                case DrawEntry::D_OBJECT: tag = SEG_OBJECT << 8 | d.index; break;
                case DrawEntry::D_EYES: case DrawEntry::D_BAR: case DrawEntry::D_BODY: tag = SEG_AGENT << 8 | d.index; break;
                case DrawEntry::D_REWARD_ROOT: case DrawEntry::D_REWARD_BOTTOM: tag = SEG_REWARD << 8 | d.index; break;
                case DrawEntry::D_MEMORY: tag = SEG_REWARD << 8 | d.index / 4; break;  // index = memory object * 4 + child
            }
            tags.push_back(tag);
        }
    if (nextSlab != slabs.size()) throw std::runtime_error("a terrain slab was not found among the drawables");
    return tags;
}

// renderView (oracle/orc_raster.hpp) with the winner's tag kept instead of shading
void segmentView(const Mat4 &view, const std::vector<Instance> &instances, const std::vector<int> &tags, int W, int H, uint16_t *seg,
                 float *depth) {
    const Projection proj(W, H);
    std::vector<SetupTri> tris;
    std::vector<int> triTag;
    for (size_t ii = 0; ii < instances.size(); ++ii) {
        const Instance &inst = instances[ii];
        const Mat4 mv = mul(view, inst.model);
        float nm[3][3];
        normalMatrix(mv, nm);
        const MeshRef mesh = meshRef(inst.mesh);
        std::vector<ClipVert> verts(size_t(mesh.nv));
        for (int v = 0; v < mesh.nv; ++v) {
            const Vec3 p{bitsToFloat(mesh.vtx[v][0]), bitsToFloat(mesh.vtx[v][1]), bitsToFloat(mesh.vtx[v][2])};
            const Vec3 nrm{bitsToFloat(mesh.vtx[v][3]), bitsToFloat(mesh.vtx[v][4]), bitsToFloat(mesh.vtx[v][5])};
            const Vec3 cam = transformPoint(mv, p);
            ClipVert &cv = verts[size_t(v)];
            cv.px = cam.x; cv.py = cam.y; cv.pz = cam.z;
            cv.cx = cam.x * proj.p00;
            cv.cy = cam.y * proj.p11;
            cv.cz = cam.z * proj.p22 + proj.p32;
            cv.cw = -cam.z;
            cv.nx = nm[0][0] * nrm.x + nm[1][0] * nrm.y + nm[2][0] * nrm.z;
            cv.ny = nm[0][1] * nrm.x + nm[1][1] * nrm.y + nm[2][1] * nrm.z;
            cv.nz = nm[0][2] * nrm.x + nm[1][2] * nrm.y + nm[2][2] * nrm.z;
        }
        for (int i = 0; i + 2 < mesh.ni; i += 3) {
            const ClipVert tri[3] = {verts[mesh.idx[i]], verts[mesh.idx[i + 1]], verts[mesh.idx[i + 2]]};
            clipAndSetup(tri, W, H, inst.color, tris);
        }
        triTag.resize(tris.size(), tags[ii]);
    }
    std::vector<float> zbuf(size_t(W) * H, 1.0f);
    std::vector<int> winner(size_t(W) * H, -1);
    std::vector<float> bary(size_t(W) * H * 3, 0.0f);
    for (int ti = 0; ti < int(tris.size()); ++ti) {
        const SetupTri &t = tris[size_t(ti)];
        int32_t minx = std::min(t.x[0], std::min(t.x[1], t.x[2])), maxx = std::max(t.x[0], std::max(t.x[1], t.x[2]));
        int32_t miny = std::min(t.y[0], std::min(t.y[1], t.y[2])), maxy = std::max(t.y[0], std::max(t.y[1], t.y[2]));
        int px0 = std::max(0, (minx - 128 + 255) >> 8), px1 = std::min(W - 1, (maxx - 128) >> 8);
        int py0 = std::max(0, (miny - 128 + 255) >> 8), py1 = std::min(H - 1, (maxy - 128) >> 8);
        bool topleft[3];
        int64_t A[3], B[3], C[3];
        for (int e = 0; e < 3; ++e) {
            const int a = (e + 1) % 3, b = (e + 2) % 3;
            const int64_t dx = int64_t(t.x[b]) - t.x[a], dy = int64_t(t.y[b]) - t.y[a];
            A[e] = dy; B[e] = -dx; C[e] = dx * t.y[a] - dy * t.x[a];
            topleft[e] = (dy == 0 && dx < 0) || dy > 0;
        }
        const float invArea = 1.0f / float(t.area);
        for (int py = py0; py <= py1; ++py)
            for (int px = px0; px <= px1; ++px) {
                const int64_t sx = int64_t(px) * 256 + 128, sy = int64_t(py) * 256 + 128;
                int64_t F[3];
                bool inside = true;
                for (int e = 0; e < 3; ++e) {
                    F[e] = A[e] * sx + B[e] * sy + C[e];
                    if (F[e] < 0 || (F[e] == 0 && !topleft[e])) { inside = false; break; }
                }
                if (!inside) continue;
                const float l0 = float(F[0]) * invArea, l1 = float(F[1]) * invArea, l2 = float(F[2]) * invArea;
                const float z = (l0 * t.z[0] + l1 * t.z[1]) + l2 * t.z[2];
                const size_t pi = size_t(py) * W + px;
                if (z <= zbuf[pi]) {
                    zbuf[pi] = z;
                    winner[pi] = ti;
                    bary[pi * 3 + 0] = l0; bary[pi * 3 + 1] = l1; bary[pi * 3 + 2] = l2;
                }
            }
    }
    for (size_t pi = 0; pi < size_t(W) * H; ++pi) {
        if (winner[pi] < 0) { seg[pi] = 0; depth[pi] = 0.0f; continue; }
        const SetupTri &t = tris[size_t(winner[pi])];
        const float k0 = bary[pi * 3 + 0] * t.rw[0], k1 = bary[pi * 3 + 1] * t.rw[1], k2 = bary[pi * 3 + 2] * t.rw[2];
        depth[pi] = 1.0f / ((k0 + k1) + k2);
        seg[pi] = uint16_t(triTag[size_t(winner[pi])]);
    }
}

}  // namespace

extern "C" {
// seg: uint16[N][h][w], depth: float[N][h][w] for the handle's current scenes (what orc_render_now draws).  0 on success, -1 when the
// tags cannot be assigned.
int orc_seg_render(void *p, uint16_t *seg, float *depth) {
    auto *v = static_cast<OrcVec *>(p);
    const size_t px = size_t(v->w) * v->h;
    try {
        for (int e = 0; e < v->numEnvs; ++e) {
            const Env &env = *v->envs[size_t(e)];
            const auto inst = env.instances();
            const auto tags = sceneTags(env);
            if (tags.size() != inst.size()) return -1;
            for (int a = 0; a < v->numAgents; ++a) {
                const size_t view = size_t(e) * v->numAgents + a;
                segmentView(env.viewMatrix(a), inst, tags, v->w, v->h, seg + view * px, depth + view * px);
            }
        }
    } catch (const std::exception &) {
        return -1;
    }
    return 0;
}
}
