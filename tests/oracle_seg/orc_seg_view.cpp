// Segmentation on the ORACLE from an arbitrary viewpoint (test infrastructure, never linked or imported by the product): orc_seg.cpp's
// segmentView for one env of an oracle vector env through a caller's view matrix at any size -- what the engine's spectator cameras
// (mv_draw_cameras) draw.  Built like orc_seg.cpp (tests/orc_seg.py), which it includes unchanged.
#include "orc_seg.cpp"

extern "C" {
// seg: uint16[h][w], depth: float[h][w] of env `env`'s current scene seen through view16 (column-major).  0 on success, -1 for an env out of
// range or when the tags cannot be assigned.
int orc_seg_render_view(void *p, int env, const float *view16, int w, int h, uint16_t *seg, float *depth) {
    auto *v = static_cast<OrcVec *>(p);
    if (env < 0 || env >= v->numEnvs) return -1;
    try {
        const Env &e = *v->envs[size_t(env)];
        const auto inst = e.instances();
        const auto tags = sceneTags(e);
        if (tags.size() != inst.size()) return -1;
        Mat4 view;
        std::memcpy(&view.c[0][0], view16, 64);
        segmentView(view, inst, tags, w, h, seg, depth);
    } catch (const std::exception &) {
        return -1;
    }
    return 0;
}
}
