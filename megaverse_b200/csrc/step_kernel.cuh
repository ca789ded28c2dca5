// K1+K2+K3: one env per warp.  Agent kinematics + capsule-vs-box/capsule collision, carry/place, reward/done, in-kernel
// episode reset from the pre-staged next level, and the per-view render inputs (view + dynamic instance matrices).
//
// Replaces (file:line under /root/reference):
//   Env::step                                   src/libs/env/src/env.cpp:83-152
//   btDiscreteDynamicsWorld::stepSimulation +
//   KinematicCharacterController                src/libs/env/src/kinematic_character_controller.cpp:156-442,509-602,625-644,753-792
//   DefaultKinematicAgent                       src/libs/env/src/agent.cpp:73-161
//   ObjectStackingComponent                     src/libs/scenarios/include/scenarios/component_object_stacking.hpp:45-198
//   FallDetectionComponent                      src/libs/scenarios/include/scenarios/component_fall_detection.hpp:33-56
//   TowerBuildingScenario::step / rewards       src/libs/scenarios/src/scenario_tower_building.cpp:179-266
//   Scenario::rewardAgent/rewardTeam            src/libs/env/include/env/scenario.hpp:251-307
//   DefaultScenario::updateUI                   src/libs/scenarios/include/scenarios/scenario_default.hpp:164-186
//   VectorEnv::step done handling               src/libs/env/src/vector_env.cpp:94-105 (reset is done in-kernel)
//   V4REnvRenderer::preDraw                     src/libs/v4r_rendering/src/v4r_env_renderer.cpp:299-336
//
// Execution model: the 32 lanes run the controller's scalar state machine redundantly on warp-uniform values held in
// shared memory; every collision query fans the env's colliders out over the lanes and reduces with warp shuffles
// (min hit fraction, lowest collider index on ties).  Static colliders and movable-object records are staged into shared
// memory with one TMA bulk copy each (cp.async.bulk + mbarrier).  Lane 0 commits state changes.
#pragma once
#include <type_traits>

#include "bzset.h"
#include "dev_math.cuh"
#include "level_set.h"
#include "mv_types.h"
#include "../../include/megaverse_b200.h"  // MV_SEG_*

namespace mvk {
using namespace dm;

constexpr float kCapsuleRadius = 0.33f;
constexpr float kCapsuleHalfHeight = 1.05f / 2;
constexpr float kAllowedCcdPenetration = 0.04f;
constexpr float kSimdEpsilon = 1.1920929e-07f;
constexpr float kMaxPenetrationDepth = 0.041f;
constexpr float kStepHeight = 0.2f;
constexpr float kGravity = 1.4f * 9.8f;
constexpr float kFallSpeed = 55.0f;
constexpr float kMaxHorizontalSpeed = 4.5f, kMaxAirSpeed = 1.0f, kNormalDeceleration = 15.0f;
constexpr float kMaxAcceleration = 35.0f + 15.0f, kMaxAirAcceleration = 3.0f, kExceedDecel = (35.0f + 15.0f) * 2;
constexpr unsigned FULL = 0xffffffffu;

struct StepParams {
    // the level arrays are indexed by level row (levelRow): [E][slots] rows with the slot ring, [level-set bank rows] with option "level_set"
    const MvLevel *levels;       // [E][slots]
    const MvBox *statics;        // [E][slots][staticCap] static layout boxes of the level slots (collider order == draw order)
    const float *staticRot;      // [E][slots][staticCap][2] MV_ROTATED boxes: local x axis in world space (ax, az)
    int staticCap;
    const uint32_t *solid;       // [E][slots][3][gridWords] planes: solid, exit terrain, lava terrain
    uint8_t *objGrid;            // [E][gridCells]
    MvEnvState *envs;            // [E]
    MvAgent *agents;             // [E*A]
    MvObject *objects;           // [E][MV_MAX_OBJECTS]
    MvInstance *instances;       // [E][instStride]
    const MvDeco *deco;          // [E][slots][decoCap] decorations of the level slots
    int decoCap, instStride;
    int32_t *instCounts;         // [E][8]
    float *views;                // [E*A][16]


    const int32_t *actions;      // [E*A]
    const float *rtable;         // [E*A][MV_R_COUNT]
    float *rewards;              // [E*A]
    uint8_t *dones;              // [E]
    float *trueObjectives;       // [E*A]
    float *hostRewards, *hostTrueObjectives;  // optional pinned host mirrors written directly by the kernel (or nullptr)
    uint8_t *hostDones;
    int32_t *hostFaults;         // pinned host word: OR of every fault bit any env ever raised (read by the host without a device round trip)
    int E, A, gridCells, gridWords;
    int forceReset;              // mv_reset(): re-initialise every env from its live level slot, no physics
    uint32_t *ready;             // [E] completion stamps polled by the geometry kernel (programmatic dependent launch)
    uint32_t readyStamp;
    const uint32_t *envOrder;  // optional [E]: warp w of the grid steps env envOrder[w] (the order in which the rasteriser will ask for the envs)
    const uint8_t *ends;         // optional [num_envs] (mv_step_device_ends): ends[env] != 0 ends the episode after this call's last tick (with 2 slots: once it has run >= 3 * repeat ticks)
    const uint8_t *active;       // optional [num_envs] (mv_step_envs, mv_step_device_active): an env whose byte is 0 runs nothing this call
    int repeat;                  // option "action_repeat": physics ticks per call (1..4), the episode stops them early
    int slots;                   // option "level_slots": level slots per env (2 or 4), one live and the rest staged in episode order
    int maxObj;                  // upper bound of n_obj over the live and staged levels (sizes the staging copy)
    // Level set (option "level_set"; levelSet == 0: off, the pointers are unused).  The level arrays are a bank of immutable rows shared by
    // the envs, MvEnvState::slot is the env's live bank row and MvEnvState::pad[0] its pick seed; an episode end chooses the next row here
    int levelSet;                // levels per scenario
    const int32_t *bankBase;     // [E] first bank row of the env's scenario: an env only ever reads rows [bankBase, bankBase + levelSet)
    int32_t *nextLevels;         // [E] the caller's choice for the env's next episode, -1 (or anything outside [0, levelSet)): the hash picks
    int32_t *levelIds;           // [E] the live level of every env stepped, within its scenario, written beside dones
    int32_t *hostLevelIds;       // optional pinned host mirror (or nullptr)
    uint32_t *prof;              // optional [E][16] per-phase cycle stamps (mv_debug_step_profile); nullptr in production
    uint8_t *doneReasons;        // [E] MV_END_* of this step, written beside dones (MV_END_NONE where dones is 0)
    uint8_t *hostDoneReasons;    // optional pinned host mirror (or nullptr)
    // optional terminal rows (option "final_obs"; nullptr: off): an env that ends at this step gets here the instance list, counts and
    // views this step would have drawn had the episode not ended.  Same layouts and instStride as instances / instCounts / views.
    MvInstance *termInstances;
    int32_t *termCounts;
    float *termViews;
    MvConsts k;
    // option "state_tensors" (nullptr: off; the stepKernel<.., true> variants only): the caller-facing rows of every env stepped, float32
    // bit copies of its state after the call (include/megaverse_b200.h has the layout): agents [E*A][16], envs [E][16], objects
    // [E][MV_MAX_OBJECTS][4], rewards [E][MV_MAX_REWARD][4].  The term* rows (with option final_obs as well) get the state an ending
    // env's terminal frame shows.
    float *stAgents, *stEnvs, *stObjects, *stRewards;
    float *termStAgents, *termStEnvs, *termStObjects, *termStRewards;
    // level set: [levelSet * banks] 0 for a row being replaced (mv_replace_levels), which no flip may land on; the host keeps at least one
    // row of every bank pickable.  Last, so that no other field moves
    const uint8_t *rowPickable;
    // option "reward_components" (nullptr: off; the stepKernel<.., .., true> variants only), each [E*A][MV_R_COUNT]: the call's reward split
    // by the shaping slot whose weight paid it, the totals of the episodes that ended in the call, and the running totals of the episodes
    // under way (include/megaverse_b200.h has the rules)
    float *rcStep, *rcEpisode, *rcRun;
    // option "autoreset" 1 or 2 (nullptr: mode 0; the stepKernel<.., .., .., 1|2> variants only): [E] MvEnvState::pad[1] after the call,
    // 1 while the env's ended episode waits for its flip, written beside dones, and its optional pinned host mirror
    uint8_t *awaiting, *hostAwaiting;
};

// option "reward_components": per warp, after the block's WarpShared records, one agent's tick columns per row -- what each shaping slot
// paid the agent this tick, [tick] like WarpShared::lastReward.  Only the stepKernel<.., .., true> variants are launched with this space
constexpr size_t kRcTickBytes = sizeof(float) * MV_MAX_AGENTS * MV_R_COUNT;

// row of the level arrays that holds slot `slot` of env `env`: the env's own ring of slots, or, with a level set, the bank row itself
template <bool kLevelSet> __device__ __forceinline__ size_t levelRow(const StepParams &P, int env, int slot) {
    return kLevelSet ? size_t(slot) : size_t(env) * P.slots + slot;
}

// One per warp.  A call runs up to P.repeat ticks (option "action_repeat") on this state and then writes its outputs once; every field
// is one of: [state] the env's state, staged once per call, carried from tick to tick and committed once; [tick] scratch rewritten by
// every tick; [call] accumulated over the call's ticks and read once after them.
struct WarpShared {
    alignas(16) MvObject objects[MV_MAX_OBJECTS];  // [state]
    alignas(16) MvAgent agents[MV_MAX_AGENTS];     // [state]
    alignas(16) MvEnvState env;                    // [state]
    alignas(8) unsigned long long mbar;            // staging barrier, once per call
    float lastReward[MV_MAX_AGENTS];               // [tick] the reward each agent is paid this tick
    int objDirty[MV_MAX_AGENTS * 2];               // [call] distinct objects picked up / put down / pushed (only tick 0 interacts)
    int nDirty;                                    // [call]
    int doneFlag;                                  // [tick] the episode ended at this tick
    uint32_t rewardDirty[4];  // [call] reward objects collected in this call (their instances need rewriting)
    uint32_t memoryNear;      // [tick] HexMemory: bit per agent that has a collectable within reach
    // [tick] this agent's collision candidates for the current tick, ascending collider index: boxes are copied here (static
    // layout boxes straight from the level in global memory, movable objects from the staged records), agents are looked
    // up live because they move within the tick
    struct Cand { float c[3]; float h[3]; int32_t kind; int32_t agent; float ax, az; } cand[MV_MAX_CAND];  // kind 2: box rotated about Y
    alignas(16) float mtx[8][16];                // cooperative 4x4 products: one element per lane (writeInstances, after the ticks)
    alignas(8) unsigned long long sweepKey[32];  // [tick] warpSweep: per live candidate, min over features of (t bits << 32 | feature)
    uint8_t sweepList[32];                       // [tick] warpSweep: lanes of the candidates that passed the swept-bounds cull
};

// ---------------------------------------------------------------- TMA (1-D bulk async copy) helpers
__device__ __forceinline__ uint32_t smemAddr(const void *p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbarInit(unsigned long long *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbarExpectTx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulkG2S(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smemAddr(dst)), "l"(src), "r"(bytes),
                 "r"(smemAddr(bar))
                 : "memory");
}
__device__ __forceinline__ void mbarWait(unsigned long long *bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smemAddr(bar)), "r"(parity)
            : "memory");
    } while (!done);
}

// ---------------------------------------------------------------- collision primitives (exact analytic; see DESIGN.md)
__device__ __forceinline__ float pointBoxDistance(V3 o, V3 H, V3 &n) {
    const V3 q = v3(fabsf(o.x) - H.x, fabsf(o.y) - H.y, fabsf(o.z) - H.z);
    if (q.x <= 0.0f && q.y <= 0.0f && q.z <= 0.0f) {
        int ax = 0;
        float best = q.x;
        if (q.y > best) { best = q.y; ax = 1; }
        if (q.z > best) { best = q.z; ax = 2; }
        n = v3(0, 0, 0);
        setComp(n, ax, comp(o, ax) < 0.0f ? -1.0f : 1.0f);
        return best;
    }
    const V3 e = v3(q.x > 0.0f ? q.x : 0.0f, q.y > 0.0f ? q.y : 0.0f, q.z > 0.0f ? q.z : 0.0f);
    const float d = sqrtf(e.x * e.x + e.y * e.y + e.z * e.z);
    n = v3(o.x < 0.0f ? -e.x : e.x, o.y < 0.0f ? -e.y : e.y, o.z < 0.0f ? -e.z : e.z);
    n = n * (1.0f / d);
    return d;
}

// Ray (capsule-axis midpoint path) against the box inflated by rho, split into its 23 boundary features so that the
// warp can test (candidate, feature) pairs in parallel: f 0..2 = the face pair of axis f (the one facing the ray),
// 3..14 = the 12 edge cylinders (axis k, then the two signs), 15..22 = the 8 corner spheres.  The closest hit of the
// whole shape is the minimum over the features with ties going to the lowest f -- the order a serial scan that only
// accepts strictly closer hits would produce.  A start point already inside the inflated shape is reported by f == 0
// alone (t = 0 along the separating normal, only when moving inwards).
constexpr int kBoxFeatures = 23;
__device__ bool rayRoundedBoxFeatureOutside(V3 o, V3 d, V3 H, float rho, int f, float &tOut, V3 &nOut);
__device__ __forceinline__ bool rayRoundedBoxFeature(V3 o, V3 d, V3 H, float rho, int f, float &tOut, V3 &nOut) {
    V3 n0;
    const float d0 = pointBoxDistance(o, H, n0);
    if (d0 - rho <= 0.0f) {
        if (f == 0 && dot(d, n0) < -kSimdEpsilon) { tOut = 0.0f; nOut = n0; return true; }
        return false;
    }
    return rayRoundedBoxFeatureOutside(o, d, H, rho, f, tOut, nOut);
}
// the feature tests proper, for a start point known to lie outside the inflated shape
__device__ bool rayRoundedBoxFeatureOutside(V3 o, V3 d, V3 H, float rho, int f, float &tOut, V3 &nOut) {
    if (f < 3) {
        const int i = f;
        const float di = comp(d, i);
        if (di == 0.0f) return false;
        const float s = di < 0.0f ? 1.0f : -1.0f;
        const float t = (s * (comp(H, i) + rho) - comp(o, i)) / di;
        if (t < 0.0f || t > 1.0f) return false;
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        const float qj = comp(o, j) + t * comp(d, j), qk = comp(o, k) + t * comp(d, k);
        if (!(fabsf(qj) <= comp(H, j) && fabsf(qk) <= comp(H, k))) return false;
        tOut = t; nOut = v3(0, 0, 0); setComp(nOut, i, s);
        return true;
    }
    if (f < 15) {
        const int e = f - 3, k = e >> 2;
        const float si = (e & 2) ? 1.0f : -1.0f, sj = (e & 1) ? 1.0f : -1.0f;
        const int i = (k + 1) % 3, j = (k + 2) % 3;
        const float di = comp(d, i), dj = comp(d, j);
        const float a = di * di + dj * dj;
        if (a == 0.0f) return false;
        const float oi = comp(o, i) - si * comp(H, i), oj = comp(o, j) - sj * comp(H, j);
        const float b = oi * di + oj * dj;
        const float c = oi * oi + oj * oj - rho * rho;
        const float disc = b * b - a * c;
        if (disc < 0.0f) return false;
        const float t = (-b - sqrtf(disc)) / a;
        if (t < 0.0f || t > 1.0f) return false;
        const float qi = oi + t * di, qj = oj + t * dj, qk = comp(o, k) + t * comp(d, k);
        if (!(si * qi >= 0.0f && sj * qj >= 0.0f && fabsf(qk) <= comp(H, k))) return false;
        tOut = t; nOut = v3(0, 0, 0);
        setComp(nOut, i, qi / rho);
        setComp(nOut, j, qj / rho);
        return true;
    }
    {
        const int e = f - 15;
        const float sx = (e & 4) ? 1.0f : -1.0f, sy = (e & 2) ? 1.0f : -1.0f, sz = (e & 1) ? 1.0f : -1.0f;
        const float a = dot(d, d);
        if (a == 0.0f) return false;
        const V3 oc = v3(o.x - sx * H.x, o.y - sy * H.y, o.z - sz * H.z);
        const float b = dot(oc, d);
        const float c = dot(oc, oc) - rho * rho;
        const float disc = b * b - a * c;
        if (disc < 0.0f) return false;
        const float t = (-b - sqrtf(disc)) / a;
        if (t < 0.0f || t > 1.0f) return false;
        const V3 q = oc + d * t;
        if (!(sx * q.x >= 0.0f && sy * q.y >= 0.0f && sz * q.z >= 0.0f)) return false;
        tOut = t; nOut = q * (1.0f / rho);
        return true;
    }
}

__device__ __forceinline__ float pointSegDistance(V3 o, float L, V3 &n) {
    const float cy = o.y < -L ? -L : (o.y > L ? L : o.y);
    const V3 e = v3(o.x, o.y - cy, o.z);
    const float d = length(e);
    if (d > 0.0f) n = e * (1.0f / d); else n = v3(1, 0, 0);
    return d;
}
__device__ bool rayCapsule(V3 o, V3 d, float L, float R, float &tOut, V3 &nOut) {
    V3 n0;
    const float d0 = pointSegDistance(o, L, n0);
    if (d0 - R <= 0.0f) {
        if (dot(d, n0) < -kSimdEpsilon) { tOut = 0.0f; nOut = n0; return true; }
        return false;
    }
    float best = 2.0f;
    V3 bestN = v3(0, 0, 0);
    {
        const float a = d.x * d.x + d.z * d.z;
        if (a != 0.0f) {
            const float b = o.x * d.x + o.z * d.z, c = o.x * o.x + o.z * o.z - R * R;
            const float disc = b * b - a * c;
            if (disc >= 0.0f) {
                const float t = (-b - sqrtf(disc)) / a;
                if (t >= 0.0f && t <= 1.0f) {
                    const float qy = o.y + t * d.y;
                    if (fabsf(qy) <= L) { best = t; bestN = v3((o.x + t * d.x) / R, 0.0f, (o.z + t * d.z) / R); }
                }
            }
        }
    }
    const float a = dot(d, d);
    if (a != 0.0f)
        for (int s = -1; s <= 1; s += 2) {
            const V3 oc = v3(o.x, o.y - s * L, o.z);
            const float b = dot(oc, d), c = dot(oc, oc) - R * R;
            const float disc = b * b - a * c;
            if (disc < 0.0f) continue;
            const float t = (-b - sqrtf(disc)) / a;
            if (t < 0.0f || t > 1.0f || t >= best) continue;
            const V3 q = oc + d * t;
            if (s * q.y >= 0.0f) { best = t; bestN = q * (1.0f / R); }
        }
    if (best > 1.0f) return false;
    tOut = best;
    nOut = bestN;
    return true;
}

// collider index space: [0,ns) statics, [ns,ns+no) objects, [ns+no, ns+no+A) agent capsules
struct ColliderView {
    const WarpShared *S;
    const MvLevel *L;
    int ns, no, A;
    int nc;  // candidates in S->cand
    // candidate j -> kind, centre, half extents
    __device__ __forceinline__ void fetch(int j, int &kind, V3 &c, V3 &h) const {
        const WarpShared::Cand &cd = S->cand[j];
        kind = cd.kind;
        if (kind != 1) { c = v3(cd.c[0], cd.c[1], cd.c[2]); h = v3(cd.h[0], cd.h[1], cd.h[2]); }
        else { const MvAgent &a = S->agents[cd.agent]; c = v3(a.pos[0], a.pos[1], a.pos[2]); h = v3(0, 0, 0); }
    }
    // boxes rotated about Y (kind 2): world <-> box frame; the local x axis in world space is (ax, 0, az)
    __device__ __forceinline__ V3 toLocal(int j, int kind, V3 p) const {
        if (kind != 2) return p;
        const float ax = S->cand[j].ax, az = S->cand[j].az;
        return v3(p.x * ax + p.z * az, p.y, p.x * -az + p.z * ax);
    }
    __device__ __forceinline__ V3 toWorld(int j, int kind, V3 n) const {
        if (kind != 2) return n;
        const float ax = S->cand[j].ax, az = S->cand[j].az;
        return v3(n.x * ax + n.z * -az, n.y, n.x * az + n.z * ax);
    }
    __device__ __forceinline__ V3 boundsExt(int j, int kind, V3 h) const {  // broadphase half extents grown by the capsule
        if (kind == 1) return v3(2.0f * kCapsuleRadius, 2.0f * (kCapsuleHalfHeight + kCapsuleRadius), 2.0f * kCapsuleRadius);
        if (kind == 2) {
            const float ax = S->cand[j].ax, az = S->cand[j].az;
            return v3((fabsf(ax) * h.x + fabsf(az) * h.z) + kCapsuleRadius, h.y + (kCapsuleHalfHeight + kCapsuleRadius), (fabsf(az) * h.x + fabsf(ax) * h.z) + kCapsuleRadius);
        }
        return v3(h.x + kCapsuleRadius, h.y + (kCapsuleHalfHeight + kCapsuleRadius), h.z + kCapsuleRadius);
    }
};

struct SweepHit { bool hit; float fraction; V3 normal; };
struct SweepReport : SweepHit { int slot, feature; };  // mv_debug_kcc: the winner's candidate slot and its feature f (0 for capsules)

// KinematicClosestNotMeConvexResultCallback over this agent's candidates.  Lanes first cull candidates against the swept
// bounds (the broadphase), then the warp tests (surviving candidate, boundary feature) pairs in parallel; each
// candidate's closest feature is found with a packed shared-memory atomicMin (t bits | feature), its lane re-evaluates
// that one feature for the exact fraction and normal, applies the callback's slope filter, and a shuffle reduction picks
// the closest candidate (ties: lowest collider index, i.e. the order a serial scan would have kept).  kReport (mv_debug_kcc only) also
// returns the winner's slot and feature.
template <bool kReport = false>
__device__ std::conditional_t<kReport, SweepReport, SweepHit> warpSweep(const ColliderView &cv, int self, V3 from, V3 to, V3 filterDir, float minSlopeDot, int lane) {
    const V3 d = to - from;
    float bt = 1.0f;
    int bi = 0x7fffffff, bf = 0;
    V3 bn = v3(0, 0, 0);
    WarpShared &S = *const_cast<WarpShared *>(cv.S);
    const float lx = from.x < to.x ? from.x : to.x, hx = from.x < to.x ? to.x : from.x;
    const float ly = from.y < to.y ? from.y : to.y, hy = from.y < to.y ? to.y : from.y;
    const float lz = from.z < to.z ? from.z : to.z, hz = from.z < to.z ? to.z : from.z;
    const float rhoBox = kCapsuleRadius - kAllowedCcdPenetration, rhoCap = 2.0f * kCapsuleRadius - kAllowedCcdPenetration;
    for (int base = 0; base < cv.nc; base += 32) {
        const int j = base + lane;  // candidates are stored in ascending collider order, so the slot is the tie-break key
        bool live = false;
        int kind = 0; V3 c = v3(0, 0, 0), h = v3(0, 0, 0);
        if (j < cv.nc) {
            cv.fetch(j, kind, c, h);
            const V3 ext = cv.boundsExt(j, kind, h);
            live = !(hx < c.x - ext.x || lx > c.x + ext.x || hy < c.y - ext.y || ly > c.y + ext.y || hz < c.z - ext.z || lz > c.z + ext.z);
        }
        if (!__ballot_sync(FULL, live)) continue;
        // a start point already inside a box's inflated shape is settled by its own lane (hit at t = 0 when moving inwards,
        // nothing otherwise); only the rest go through the feature tests
        bool needFeatures = live;
        if (live) {
            unsigned long long key0 = ~0ull;
            if (kind != 1) {
                V3 n0;
                const float d0 = pointBoxDistance(cv.toLocal(j, kind, from - c), v3(h.x, h.y + kCapsuleHalfHeight, h.z), n0);
                if (d0 - rhoBox <= 0.0f) {
                    needFeatures = false;
                    if (dot(cv.toLocal(j, kind, d), n0) < -kSimdEpsilon) key0 = 0ull;  // t = 0, feature 0
                }
            }
            S.sweepKey[lane] = key0;
        }
        const unsigned m = __ballot_sync(FULL, needFeatures);
        const int nlive = __popc(m);
        if (needFeatures) S.sweepList[__popc(m & ((1u << lane) - 1u))] = uint8_t(lane);
        __syncwarp();
        // feature-major item order: neighbouring lanes run the same kind of test on different candidates
        const float invLive = 1.0f / float(nlive > 0 ? nlive : 1);
        for (int item = lane; item < nlive * kBoxFeatures; item += 32) {
            int f = int((float(item) + 0.5f) * invLive);
            int q = item - f * nlive;
            if (q < 0) { f -= 1; q += nlive; } else if (q >= nlive) { f += 1; q -= nlive; }
            const int src = S.sweepList[q];
            int k2; V3 c2, h2;
            cv.fetch(base + src, k2, c2, h2);
            float t; V3 nn; bool hit = false;
            if (k2 != 1) hit = rayRoundedBoxFeatureOutside(cv.toLocal(base + src, k2, from - c2), cv.toLocal(base + src, k2, d), v3(h2.x, h2.y + kCapsuleHalfHeight, h2.z), rhoBox, f, t, nn);
            else if (f == 0) hit = rayCapsule(from - c2, d, 2.0f * kCapsuleHalfHeight, rhoCap, t, nn);
            if (hit) atomicMin(&S.sweepKey[src], (static_cast<unsigned long long>(__float_as_uint(t + 0.0f)) << 32) | unsigned(f));
        }
        __syncwarp();
        if (live) {
            const unsigned long long key = S.sweepKey[lane];
            if (key != ~0ull) {
                float t; V3 nn;
                if (kind != 1) {
                    rayRoundedBoxFeature(cv.toLocal(j, kind, from - c), cv.toLocal(j, kind, d), v3(h.x, h.y + kCapsuleHalfHeight, h.z), rhoBox, int(key & 31u), t, nn);
                    nn = cv.toWorld(j, kind, nn);
                } else rayCapsule(from - c, d, 2.0f * kCapsuleHalfHeight, rhoCap, t, nn);
                if (t < bt && !(dot(filterDir, nn) < minSlopeDot)) {
                    bt = t; bi = j; bn = nn;
                    if constexpr (kReport) bf = int(key & 31u);
                }
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const float ot = __shfl_xor_sync(FULL, bt, off);
        const int oi = __shfl_xor_sync(FULL, bi, off);
        const float ox = __shfl_xor_sync(FULL, bn.x, off), oy = __shfl_xor_sync(FULL, bn.y, off), oz = __shfl_xor_sync(FULL, bn.z, off);
        if constexpr (kReport) {
            const int of = __shfl_xor_sync(FULL, bf, off);
            if (ot < bt || (ot == bt && oi < bi)) bf = of;
        }
        if (ot < bt || (ot == bt && oi < bi)) { bt = ot; bi = oi; bn = v3(ox, oy, oz); }
    }
    std::conditional_t<kReport, SweepReport, SweepHit> r;
    r.hit = bi != 0x7fffffff;
    r.fraction = r.hit ? bt : 1.0f;
    r.normal = bn;
    if constexpr (kReport) { r.slot = bi; r.feature = bf; }
    return r;
}

// first collider (index order) penetrating deeper than maxPenetrationDepth; returns push-out delta (and, when slotOut is given, that
// collider's candidate slot: mv_debug_kcc only)
template <bool kReport = false>
__device__ bool warpRecover(const ColliderView &cv, int self, V3 p, V3 &delta, int lane, int *slotOut = nullptr) {
    for (int base = 0; base < cv.nc; base += 32) {
        const int j = base + lane;
        bool pen = false;
        V3 dl = v3(0, 0, 0);
        if (j < cv.nc) {
            int kind; V3 c, h;
            cv.fetch(j, kind, c, h);
            V3 nn;
            float dist;
            if (kind != 1) { dist = pointBoxDistance(cv.toLocal(j, kind, p - c), v3(h.x, h.y + kCapsuleHalfHeight, h.z), nn) - kCapsuleRadius; nn = cv.toWorld(j, kind, nn); }
            else dist = pointSegDistance(p - c, 2.0f * kCapsuleHalfHeight, nn) - 2.0f * kCapsuleRadius;
            if (dist < -kMaxPenetrationDepth) { pen = true; dl = nn * (-dist); }
        }
        const unsigned m = __ballot_sync(FULL, pen);
        if (m) {
            const int src = __ffs(m) - 1;
            delta = v3(__shfl_sync(FULL, dl.x, src), __shfl_sync(FULL, dl.y, src), __shfl_sync(FULL, dl.z, src));
            if constexpr (kReport) *slotOut = base + src;
            return true;
        }
    }
    return false;
}

// ---------------------------------------------------------------- kinematic character controller (uniform across lanes)
struct Kcc {
    V3 pos, hvel, jumpAxis, cur, tgt;
    float vvel, voff, stepOff, jumpSpeed;
    bool wasOnGround, wasJumping;
#ifdef MV_KCC_COUNTERS
    uint32_t dbg[4] = {0, 0, 0, 0};  // sweeps, recovers, cycles in sweeps, cycles in recovers
#endif
    __device__ __forceinline__ bool onGround() const { return (fabsf(vvel) < kSimdEpsilon) && (fabsf(voff) < kSimdEpsilon); }
};

__device__ __forceinline__ V3 lerp3(V3 a, V3 b, float rt) {  // btVector3::setInterpolate3
    const float s = 1.0f - rt;
    return v3(s * a.x + rt * b.x, s * a.y + rt * b.y, s * a.z + rt * b.z);
}

__device__ void kccSetAcceleration(Kcc &k, V3 acc, float dt) {
    const bool isOnGround = k.onGround();
    const float accelerationMagnitude = length(acc);
    const float currMax = isOnGround ? kMaxAcceleration : kMaxAirAcceleration;
    if (!(length2(acc) < kSimdEpsilon * kSimdEpsilon)) acc = acc * (currMax / accelerationMagnitude);
    if (isOnGround) {
        k.hvel = k.hvel + acc * dt;
        const float sp = length(k.hvel);
        if (sp > kMaxHorizontalSpeed) {
            const float dv = kExceedDecel * dt;
            if (sp - dv > kMaxHorizontalSpeed) k.hvel = k.hvel * ((sp - dv) / sp);
            else k.hvel = k.hvel * (kMaxHorizontalSpeed / sp);
        }
    } else {
        const float sp = length(k.hvel);
        const V3 nv = k.hvel + acc * dt;
        const float nsp = length(nv);
        if (nsp <= kMaxAirSpeed || nsp < sp) k.hvel = nv;
    }
}

__device__ bool kccRecover(Kcc &k, const ColliderView &cv, int self, int lane) {
    k.cur = k.pos;
    V3 delta;
#ifdef MV_KCC_COUNTERS
    const long long tr0 = clock64();
#endif
    const bool pen = warpRecover(cv, self, k.cur, delta, lane);
#ifdef MV_KCC_COUNTERS
    k.dbg[1]++; k.dbg[3] += uint32_t(clock64() - tr0);
#endif
    if (pen) k.cur = k.cur + delta;
    k.pos = k.cur;
    return pen;
}

#ifdef MV_KCC_COUNTERS
#define warpSweep(...) ([&] { const long long ts0 = clock64(); const SweepHit r_ = warpSweep(__VA_ARGS__); k.dbg[0]++; k.dbg[2] += uint32_t(clock64() - ts0); return r_; }())
#endif
__device__ void kccPlayerStep(Kcc &k, const ColliderView &cv, int self, float dt, float maxSlopeCos, int lane) {
    const V3 up = v3(0, 1, 0);
    k.cur = k.pos;
    k.tgt = k.cur;
    const V3 original = k.cur;
    k.wasOnGround = k.onGround();
    k.vvel -= kGravity * dt;
    if (k.vvel > 0.0f && k.vvel > k.jumpSpeed) k.vvel = k.jumpSpeed;
    if (k.vvel < 0.0f && fabsf(k.vvel) > fabsf(kFallSpeed)) k.vvel = -fabsf(kFallSpeed);
    k.voff = k.vvel * dt;
    {  // stepUp
        float stepH = 0.0f;
        if (k.vvel < 0.0f) stepH = kStepHeight;
        const V3 start = k.cur;
        k.tgt = k.cur + up * stepH + k.jumpAxis * (k.voff > 0.f ? k.voff : 0.f);
        k.cur = k.tgt;
        const SweepHit cb = warpSweep(cv, self, start, k.tgt, -up, maxSlopeCos, lane);
        if (cb.hit) {
            if (dot(cb.normal, up) > 0.0f) {
                k.stepOff = stepH * cb.fraction;
                k.cur = lerp3(k.cur, k.tgt, cb.fraction);
            }
            k.pos = k.cur;
            int loops = 0;
            while (kccRecover(k, cv, self, lane)) {
                loops++;
                if (loops > 4) break;
            }
            k.tgt = k.pos;
            k.cur = k.tgt;
            if (k.voff > 0) { k.voff = 0.0f; k.vvel = 0.0f; k.stepOff = kStepHeight; }
        } else {
            k.stepOff = stepH;
            k.cur = k.tgt;
        }
    }
    {  // stepForwardAndStrafe
        const V3 hv = k.hvel;
        k.tgt = k.cur + hv * dt;
        int maxIter = 10;
        while (maxIter-- > 0) {
            const V3 sweepDirNegative = k.cur - k.tgt;
            SweepHit cb;
            cb.hit = false; cb.fraction = 1.0f; cb.normal = v3(0, 0, 0);
            const bool same = k.cur.x == k.tgt.x && k.cur.y == k.tgt.y && k.cur.z == k.tgt.z;
            if (!same) cb = warpSweep(cv, self, k.cur, k.tgt, sweepDirNegative, 0.0f, lane);
            if (cb.hit) {
                {  // updateTargetPositionBasedOnCollision
                    V3 md = k.tgt - k.cur;
                    const float ml = length(md);
                    if (ml > kSimdEpsilon) {
                        md = btNormalized(md);
                        const V3 par = cb.normal * dot(md, cb.normal);
                        const V3 perp = md - par;
                        k.tgt = k.cur;
                        k.tgt = k.tgt + perp * ml;
                        k.tgt = k.tgt + par * (ml * cb.fraction);
                    }
                }
                V3 cd = k.tgt - k.cur;
                const float d2 = length2(cd);
                if (d2 > 0.0001f) {
                    cd = btNormalized(cd);
                    if (dot(cd, hv) <= 0.0f) { k.tgt = k.cur; break; }
                } else { k.tgt = k.cur; break; }
            } else break;
        }
        k.cur = k.tgt;
    }
    {  // stepDown
        float down = (k.vvel < 0.f ? -k.vvel : 0.f);
        if (down > 0.0f && down > kFallSpeed && (k.wasOnGround || !k.wasJumping)) down = kFallSpeed;
        const V3 drop = up * (k.stepOff + down * dt);
        k.tgt = k.tgt - drop;
        const SweepHit cb = warpSweep(cv, self, k.cur, k.tgt, up, maxSlopeCos, lane);
        if (cb.hit) {
            k.cur = lerp3(k.cur, k.tgt, cb.fraction);
            k.vvel = 0.0f; k.voff = 0.0f; k.wasJumping = false;
        } else k.cur = k.tgt;
    }
    k.pos = k.cur;
    k.hvel = (k.cur - original) * (1.0f / dt);
    k.hvel.y = 0;
    int loops = 0;
    while (kccRecover(k, cv, self, lane)) {
        loops++;
        if (loops > 4) break;
    }
    const float sp = length(k.hvel);
    if (k.onGround()) {
        if (sp - kNormalDeceleration * dt < 0) k.hvel = v3(0, 0, 0);
        else k.hvel = k.hvel * ((sp - kNormalDeceleration * dt) / sp);
    }
}

#ifdef MV_KCC_COUNTERS
#undef warpSweep
#endif

// ---------------------------------------------------------------- per-step collision candidates
// The box an agent at p can move in within one step (0.2 step-up + jump, <= 55/15 fall, <= 5 push-outs): colliders whose bounds miss it
// are left out of the step's sweeps and recoveries.  An agent that ends the step within 0.5 of its faces sets MV_FAULT_ENVELOPE.
__device__ __forceinline__ V3 envelopeLo(V3 p) { return v3(p.x - 3.0f, p.y - 6.0f, p.z - 3.0f); }
__device__ __forceinline__ V3 envelopeHi(V3 p) { return v3(p.x + 3.0f, p.y + 3.0f, p.z + 3.0f); }
__device__ __forceinline__ bool leftEnvelope(V3 envLo, V3 envHi, V3 p) {
    return p.x < envLo.x + 0.5f || p.x > envHi.x - 0.5f || p.y < envLo.y + 0.5f || p.y > envHi.y - 0.5f || p.z < envLo.z + 0.5f || p.z > envHi.z - 0.5f;
}

// Agent i's candidate colliders for the whole step into S.cand, in ascending collider order: everything whose bounds (grown by the
// capsule) reach the envelope [envLo, envHi].  Statics come from global memory, objects and agents from S.  Returns the count, at most
// MV_MAX_CAND; more sets MV_FAULT_CAND_OVERFLOW in S.env.faults.  slotCollider, when given, receives each slot's collider index.
__device__ __forceinline__ int gatherCandidates(WarpShared &S, const MvBox *statics, const float *staticRot, int nsPre, int ns, int no, int A, int i,
                                                V3 envLo, V3 envHi, int lane, int16_t *slotCollider = nullptr) {
    int nc = 0;
    const int n = ns + no + A;
    for (int base = 0; base < n; base += 32) {
        const int ci = base + lane;
        bool keep = false;
        int kind = 0, agentIdx = 0;
        float rax = 1.0f, raz = 0.0f;
        V3 c = v3(0, 0, 0), h = v3(0, 0, 0);
        // collider order (= the reference's creation order, which decides ties): the first nsPre static boxes,
        // the movable objects, the remaining static boxes, the agents
        if (ci < nsPre || (ci >= nsPre + no && ci < ns + no)) {
            const int si = ci < nsPre ? ci : ci - no;
            const MvBox &sb = statics[si];  // global memory (L2 resident): scanned once per agent per step
            if (sb.flags & MV_SOLID) {
                keep = true; c = v3(sb.c[0], sb.c[1], sb.c[2]); h = v3(sb.h[0], sb.h[1], sb.h[2]);
                if (sb.flags & MV_ROTATED) { kind = 2; rax = staticRot[size_t(si) * 2]; raz = staticRot[size_t(si) * 2 + 1]; }
            }
        } else if (ci < nsPre + no) {
            const MvObject &ob = S.objects[ci - nsPre];
            if (ob.enabled) { keep = true; c = v3(ob.col_c[0], ob.col_c[1], ob.col_c[2]); h = v3(ob.col_h[0], ob.col_h[1], ob.col_h[2]); }
        } else if (ci < n && ci - ns - no != i) {
            agentIdx = ci - ns - no;
            const MvAgent &oa = S.agents[agentIdx];
            keep = true; kind = 1; c = v3(oa.pos[0], oa.pos[1], oa.pos[2]);
        }
        if (keep) {
            // agents may move up to an envelope of their own within this step: give capsules the same slack
            V3 ext = kind != 1 ? v3(h.x + kCapsuleRadius, h.y + (kCapsuleHalfHeight + kCapsuleRadius), h.z + kCapsuleRadius)
                               : v3(2.0f * kCapsuleRadius + 3.0f, 2.0f * (kCapsuleHalfHeight + kCapsuleRadius) + 6.0f, 2.0f * kCapsuleRadius + 3.0f);
            if (kind == 2) { ext.x = (fabsf(rax) * h.x + fabsf(raz) * h.z) + kCapsuleRadius; ext.z = (fabsf(raz) * h.x + fabsf(rax) * h.z) + kCapsuleRadius; }
            keep = !(envHi.x < c.x - ext.x || envLo.x > c.x + ext.x || envHi.y < c.y - ext.y || envLo.y > c.y + ext.y ||
                     envHi.z < c.z - ext.z || envLo.z > c.z + ext.z);
        }
        const unsigned m = __ballot_sync(FULL, keep);
        const int slotC = nc + __popc(m & ((1u << lane) - 1u));
        if (keep && slotC < MV_MAX_CAND) {
            WarpShared::Cand &cd = S.cand[slotC];
            cd.c[0] = c.x; cd.c[1] = c.y; cd.c[2] = c.z; cd.h[0] = h.x; cd.h[1] = h.y; cd.h[2] = h.z; cd.kind = kind; cd.agent = agentIdx; cd.ax = rax; cd.az = raz;
            if (slotCollider) slotCollider[slotC] = int16_t(ci);
        }
        nc += __popc(m);
    }
    if (nc > MV_MAX_CAND) { nc = MV_MAX_CAND; S.env.faults |= MV_FAULT_CAND_OVERFLOW; }
    __syncwarp();
    return nc;
}


// ---------------------------------------------------------------- helpers on shared state
__device__ __forceinline__ M4 loadM4(const float *p) { M4 m;
#pragma unroll
    for (int i = 0; i < 16; ++i) m.c[i] = p[i];
    return m; }
__device__ __forceinline__ void storeM4(float *p, const M4 &m) {
#pragma unroll
    for (int i = 0; i < 16; ++i) p[i] = m.c[i]; }
__device__ __forceinline__ M4 pickupLocal() { return mul4(translation4(v3(0.0f, -0.44f, -1.0f)), identity4()); }

// DefaultKinematicAgent::updateTransform (agent.cpp:73-98).  Returns false (and leaves object_t) on NaN.
__device__ bool updateTransform(MvAgent &a, M4 &out) {
    // btMatrix3x3::getRotation
    const float *m = a.basis;
    const float trace = m[0] + m[4] + m[8];
    float t[4];
    if (trace > 0.0f) {
        float s = sqrtf(trace + 1.0f);
        t[3] = s * 0.5f;
        s = 0.5f / s;
        t[0] = (m[7] - m[5]) * s;
        t[1] = (m[2] - m[6]) * s;
        t[2] = (m[3] - m[1]) * s;
    } else {
        const int i = m[0] < m[4] ? (m[4] < m[8] ? 2 : 1) : (m[0] < m[8] ? 2 : 0);
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        float s = sqrtf(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0f);
        t[i] = s * 0.5f;
        s = 0.5f / s;
        t[3] = (m[k * 3 + j] - m[j * 3 + k]) * s;
        t[j] = (m[j * 3 + i] + m[i * 3 + j]) * s;
        t[k] = (m[k * 3 + i] + m[i * 3 + k]) * s;
    }
    V3 position = v3(a.pos[0], a.pos[1], a.pos[2]);
    V3 axis;
    {
        const float s2 = 1.0f - t[3] * t[3];
        if (s2 < 10.0f * kSimdEpsilon) axis = v3(1, 0, 0);
        else { const float s = 1.0f / sqrtf(s2); axis = v3(t[0] * s, t[1] * s, t[2] * s); }
    }
    const V3 na = mgNormalized(axis);
    const float wq = t[3] < -1.0f ? -1.0f : (t[3] > 1.0f ? 1.0f : t[3]);  // btAcos clamps (btScalar.h)
    const float rotation = 2.0f * cracos(wq);
    if (isnan(position.x) || isnan(position.y) || isnan(position.z) || isnan(rotation)) return false;
    if (isnan(na.x) || isnan(na.y) || isnan(na.z)) return false;
    position = position + v3(0, 0.05f, 0.0f);
    out = mul4(translation4(position), mul4(rotation4(rotation, na), identity4()));
    return true;
}

__device__ __forceinline__ int gridIndex(const MvLevel &L, int x, int y, int z) {
    const int gx = x - L.grid_org[0], gy = y - L.grid_org[1], gz = z - L.grid_org[2];
    if (gx < 0 || gy < 0 || gz < 0 || gx >= L.grid_dim[0] || gy >= L.grid_dim[1] || gz >= L.grid_dim[2]) return -1;
    return (gx * L.grid_dim[1] + gy) * L.grid_dim[2] + gz;
}
// voxel_grid.hpp:18-21,144-149 with origin 0, voxelSize 1
__device__ __forceinline__ void toVoxel(V3 v, int &x, int &y, int &z) {
    x = int(lroundf(floorf((v.x - 0.0f) / 1.0f))); y = int(lroundf(floorf((v.y - 0.0f) / 1.0f))); z = int(lroundf(floorf((v.z - 0.0f) / 1.0f)));
}

__device__ __forceinline__ bool inBuildingZone(const MvLevel &L, int x, int z) {
    return x >= L.bz_min[0] && x < L.bz_max[0] && z >= L.bz_min[2] && z < L.bz_max[2];
}
__device__ __forceinline__ float towerCoeff(float height) {  // buildingRewardCoeffForHeight
    float res = height * 0.05f;
    const float p2 = ldexpf(1.0f, int(height));  // powf(2, height) for integral heights, exact
    const float v = 0.05f * p2;
    res += v < 20.0f ? v : 20.0f;
    return res;
}
__device__ float towerReward(const MvEnvState &e) {
    float r = 0.0f;
    for (int i = 0; i < e.bz_count; ++i) r += towerCoeff(float(e.bz_items[i][1]));
    return r;
}

// RigidBody::syncPose for an object resting in the scene (identity parent): centre = t + collisionOffset,
// half = scaling * collisionScale (physics.hpp:69-74); the class selects the pair the scenario set on the body
__device__ __forceinline__ void syncPoseScene(MvObject &o) {
    const int cls = MV_OBJ_COLCLASS(o.meta);
    const float offY = cls == 0 ? -0.05f : (cls == 4 ? 0.6f : 0.0f);
    const float sx = (cls == 0 || cls == 4) ? 1.15f : 1.0f, sy = cls == 0 ? 1.15f : (cls == 2 ? 0.5f : (cls == 3 ? 2.0f : (cls == 4 ? 3.0f : 1.0f))), sz = sx;
    o.col_c[0] = o.t[0] + 0.0f; o.col_c[1] = o.t[1] + offY; o.col_c[2] = o.t[2] + 0.0f;
    o.col_h[0] = sqrtf(o.s[0] * o.s[0] + 0.0f * 0.0f + 0.0f * 0.0f) * sx;
    o.col_h[1] = sqrtf(0.0f * 0.0f + o.s[1] * o.s[1] + 0.0f * 0.0f) * sy;
    o.col_h[2] = sqrtf(0.0f * 0.0f + 0.0f * 0.0f + o.s[2] * o.s[2]) * sz;
}

// RearrangeScenario::countMatchingObjects (scenario_rearrange.cpp:134-149): resting objects whose voxel offset from the work
// centre equals a target item of the same shape and colour
__device__ int rearrangeCountMatches(const WarpShared &S, const MvLevel &L) {
    int matches = 0;
    for (int oi = 0; oi < L.n_obj; ++oi) {
        const MvObject &ob = S.objects[oi];
        if (ob.parent >= 0) continue;  // pickedUp
        const int x = int(lroundf(floorf(ob.t[0]))), y = int(lroundf(floorf(ob.t[1]))), z = int(lroundf(floorf(ob.t[2])));
        const int ox = x - L.work_center[0], oy = y - L.work_center[1], oz = z - L.work_center[2];
        for (int q = 0; q < L.n_arr; ++q)
            if (L.arr[q][0] == MV_OBJ_MESH(ob.meta) && L.arr[q][1] == ob.color && L.arr[q][2] == ox && L.arr[q][3] == oy && L.arr[q][4] == oz) { ++matches; break; }
    }
    return matches;
}

// ---------------------------------------------------------------- episode (re)initialisation from a level slot
__device__ void resetEnv(WarpShared &S, const MvLevel &L, uint8_t *objGrid, int A, int lane) {
    // voxel -> object map: only the words that cover this level's grid.  Every reader bounds its index by grid_dim (gridIndex), so the
    // bytes beyond it are never read; the product fits the scenario's capacity (the generator checks it) and the row pitch is a
    // multiple of 128 cells, so rounding up to whole words stays inside the row.
    {
        uint32_t *g32 = reinterpret_cast<uint32_t *>(objGrid);
        const int words = (L.grid_dim[0] * L.grid_dim[1] * L.grid_dim[2] + 3) / 4;
        for (int i = lane; i < words; i += 32) g32[i] = 0xffffffffu;
        __syncwarp();
    }
    for (int i = lane; i < L.n_obj; i += 32) {
        MvObject &o = S.objects[i];
        const MvObjInit &oi = L.obj_init[i];
        const int x = oi.voxel[0], y = oi.voxel[1], z = oi.voxel[2];
        o.t[0] = oi.pos[0]; o.t[1] = oi.pos[1]; o.t[2] = oi.pos[2];
        o.s[0] = oi.scale[0]; o.s[1] = oi.scale[1]; o.s[2] = oi.scale[2];
        o.parent = -1; o.enabled = 1; o.color = oi.color; o.meta = oi.meta;
        syncPoseScene(o);
        const int gi = gridIndex(L, x, y, z);
        if (gi >= 0) objGrid[gi] = uint8_t(i);
    }
    for (int i = lane; i < A; i += 32) {
        MvAgent &a = S.agents[i];
        for (int k = 0; k < 3; ++k) { a.pos[k] = L.spawn_pos[i][k]; a.hvel[k] = 0.0f; }
        for (int k = 0; k < 9; ++k) a.basis[k] = L.spawn_basis[i][k];
        a.vvel = 0; a.voff = 0; a.step_off = 0; a.jump_speed = 10.0f;
        a.jump_axis[0] = 0; a.jump_axis[1] = 1; a.jump_axis[2] = 0;
        a.cur_x = 0.0f;
        storeM4(a.cam_local, mul4(translation4(v3(0, 0.41f, 0)), identity4()));
        a.bar_scale[0] = 0.24f; a.bar_scale[1] = float(0.0015); a.bar_scale[2] = float(0.001);
        a.total_reward = 0.0f;
        a.was_on_ground = 0; a.was_jumping = 0; a.carrying = -1; a.picked_up = 0; a.visited_bz = 0;
        M4 ot;
        if (updateTransform(a, ot)) storeM4(a.object_t, ot); else storeM4(a.object_t, identity4());
    }
    __syncwarp();
    if (lane == 0) {
        MvEnvState &e = S.env;
        e.episode_sec = 0.0f; e.num_frames = 0; e.highest_tower = 0;
        e.solved = 0; e.reached_exit = 0u; e.positive_collected = 0;
        for (int w = 0; w < 4; ++w) { const int nb = L.n_reward - 32 * w; e.reward_alive[w] = nb >= 32 ? 0xffffffffu : (nb > 0 ? ((1u << nb) - 1u) : 0u); }
        mvBzClear(e);
        if (L.scenario == MV_SCENARIO_TOWER) {
            for (int i = 0; i < L.n_obj; ++i) {
                const int x = L.obj_init[i].voxel[0], y = L.obj_init[i].voxel[1], z = L.obj_init[i].voxel[2];
                if (inBuildingZone(L, x, z)) mvBzInsert(e, x, y, z);
            }
            e.bz_reward = towerReward(e);
        } else e.bz_reward = 0.0f;
        if (L.scenario == MV_SCENARIO_REARRANGE) e.reached_exit = uint32_t(rearrangeCountMatches(S, L));  // maxMatchingObjects at episode start
    }
    __syncwarp();
}

// ---------------------------------------------------------------- cooperative 4x4 algebra: one output element per lane
// Same operation order per element as mul4 / inverted4 (dev_math.cuh), so results are bit-identical to the serial forms;
// sixteen lanes produce one matrix, the warp two at a time.
__device__ __forceinline__ float mul4Elem(const float *a, const float *b, int e) {
    const int row = e & 3, col = e >> 2;
    float acc = 0.0f;
#pragma unroll
    for (int pos = 0; pos < 4; ++pos) acc += a[pos * 4 + row] * b[col * 4 + pos];
    return acc;
}
__device__ __forceinline__ float det3skipP(const float *m, int skipCol, int skipRow) {
#define MV_E(ci, ri) m[((ci) + ((ci) >= skipCol)) * 4 + ((ri) + ((ri) >= skipRow))]
    return MV_E(0, 0) * ((MV_E(1, 1) * MV_E(2, 2)) - (MV_E(2, 1) * MV_E(1, 2))) - MV_E(0, 1) * (MV_E(1, 0) * MV_E(2, 2) - MV_E(2, 0) * MV_E(1, 2)) +
           MV_E(0, 2) * (MV_E(1, 0) * MV_E(2, 1) - MV_E(2, 0) * MV_E(1, 1));
#undef MV_E
}
__device__ __forceinline__ float cofactor4P(const float *m, int col, int row) { return (((row + col) & 1) ? -1 : 1) * det3skipP(m, col, row); }
__device__ __forceinline__ float inv4Elem(const float *m, int e) {
    const int row = e & 3, col = e >> 2;
    float d = 0.0f;
#pragma unroll
    for (int c = 0; c < 4; ++c) d += m[c * 4] * cofactor4P(m, c, 0);
    return cofactor4P(m, row, col) / d;
}
// T(t) * S(s) element e (see tsMatrix)
__device__ __forceinline__ float tsElem(float tx, float ty, float tz, float sx, float sy, float sz, int e) {
    return e == 0 ? sx : e == 5 ? sy : e == 10 ? sz : e == 12 ? tx : e == 13 ? ty : e == 14 ? tz : e == 15 ? 1.0f : 0.0f;
}

// ---------------------------------------------------------------- render inputs (K3): instance list + view matrices
// Model matrices are the drawables' absoluteTransformationMatrix() (v4r_env_renderer.cpp:52-55), which Magnum evaluates as
// compose(parent.absoluteTransformation(), transformation()) -- left to right from the scene root (SceneGraph/Object.hpp:114-117).
// tag: the drawable's segmentation class and index, MV_SEG_* << 8 | index (the rasteriser's option "segmentation" draws it)
__device__ __forceinline__ int segTag(int cls, int index) { return cls << 8 | index; }
__device__ __forceinline__ void putInstance(MvInstance &d, const M4 &m, int mesh, int color, int tag) {
    storeM4(d.model, m);
    d.mesh = mesh; d.color = color; d.pad[0] = tag; d.pad[1] = 0;
}
// T(t) * (S(s) * I) built directly: every product in the generic 4x4 chain is x*1 or x*0 and every partial sum adds +0, so
// this is bit-identical to the multiplied-out matrix (scale and translation components are positive or zero terms)
__device__ __forceinline__ M4 tsMatrix(V3 t, V3 sc) {
    M4 m;
#pragma unroll
    for (int i = 0; i < 16; ++i) m.c[i] = 0.0f;
    m.c[0] = sc.x; m.c[5] = sc.y; m.c[10] = sc.z; m.c[12] = t.x; m.c[13] = t.y; m.c[14] = t.z; m.c[15] = 1.0f;
    return m;
}

__device__ void writeInstances(const WarpShared &S, const MvLevel &L, const MvBox *statics, const MvDeco *deco, MvInstance *inst, int32_t *counts, float *views, int A, bool writeStatic, int lane) {
    // static part (every slot is precomputed by the host in draw order): opaque layout boxes, terrain slabs, decorations
    if (writeStatic) {
        for (int i = lane; i < L.n_static; i += 32) {
            const MvBox &b = statics[i];
            if (!(b.flags & MV_OPAQUE)) continue;
            putInstance(inst[b.flags >> 8], tsMatrix(v3(b.c[0], b.c[1], b.c[2]), v3(b.h[0], b.h[1], b.h[2])), 0, b.color, segTag(MV_SEG_STATIC, 0));
        }
        for (int i = lane; i < L.n_terrain; i += 32)  // type is one TerrainType bit
            putInstance(inst[L.slot_terrain + i], loadM4(L.terrain[i].model), 0, L.terrain[i].color, segTag(MV_SEG_TERRAIN, __ffs(L.terrain[i].type) - 1));
        for (int i = lane; i < L.n_deco; i += 32) putInstance(inst[deco[i].slot], loadM4(deco[i].model), deco[i].mesh, deco[i].color, segTag(MV_SEG_STATIC, 0));
    }
    const int no = L.n_obj;
    // movable objects: everything at reset, afterwards only what can have moved -- carried objects (they follow their
    // agent's camera) and the objects picked up / put down this step
    const int nTouch = writeStatic ? no : A + S.nDirty;
    for (int idx = lane; idx < nTouch; idx += 32) {
        const int i = writeStatic ? idx : (idx < A ? S.agents[idx].carrying : S.objDirty[idx - A]);
        if (i < 0) continue;
        const MvObject &o = S.objects[i];
        M4 m = tsMatrix(v3(o.t[0], o.t[1], o.t[2]), v3(o.s[0], o.s[1], o.s[2]));
        if (o.parent >= 0) {
            const MvAgent &a = S.agents[o.parent];
            m = mul4(mul4(mul4(loadM4(a.object_t), loadM4(a.cam_local)), pickupLocal()), m);  // left to right, as absoluteTransformation()
        }
        putInstance(inst[MV_OBJ_SLOT(o.meta)], m, MV_OBJ_MESH(o.meta), o.color, segTag(MV_SEG_OBJECT, i));
    }
    // per agent: view matrix, eyes, HUD bar, body.  Every chain is associated the way Magnum's absoluteTransformation()
    // recursion does it (SceneGraph/Object.hpp:114-117): from the root, left to right -- ((objT * cam) * ui) * anchor) * bar.
    // Products are formed cooperatively (sixteen lanes per matrix, two matrices per round):
    //   r1  T3 = objT * cam              body instance = objT * body
    //   r2  eyes instance = T3 * eyes    T1 = T3 * ui
    //   r3  view = inverse(T3)           T2 = T1 * anchor
    //   r4                               bar instance = T2 * bar
    {
        float (*T)[16] = const_cast<float (*)[16]>(S.mtx);
        const int half = lane >> 4, e = lane & 15;
        const float eyesE = tsElem(0.0f, 0.0f, -0.19f, 0.25f, 0.12f, 0.2f, e), uiE = tsElem(0, 0, -0.2f, 1, 1, 1, e);
        const float anchorE = tsElem(0, -0.131f, 0, 1, 1, 1, e), bodyE = tsElem(0, 0.09f, 0, 0.35f, 0.36f, 0.35f, e);
        // constant locals: slots 5 (eyes), 6 (ui), 7 (anchor), 0 (body)
        if (half == 0) { T[5][e] = eyesE; T[6][e] = uiE; } else { T[7][e] = anchorE; T[0][e] = bodyE; }
        for (int i = 0; i < A; ++i) {
            const MvAgent &a = S.agents[i];
            const float *objT = a.object_t, *cam = a.cam_local;
            if (half == 1) T[4][e] = tsElem(0, 0, 0, a.bar_scale[0], a.bar_scale[1], a.bar_scale[2], e);  // scaling4(bar)
            __syncwarp();
            {  // r1
                if (half == 0) T[3][e] = mul4Elem(objT, cam, e);
                else inst[L.slot_body + i].model[e] = mul4Elem(objT, T[0], e);
            }
            __syncwarp();
            {  // r2
                const float v = half == 0 ? mul4Elem(T[3], T[5], e) : mul4Elem(T[3], T[6], e);
                if (half == 0) inst[L.slot_eyes + i].model[e] = v; else T[1][e] = v;
            }
            __syncwarp();
            {  // r3
                if (half == 0) views[i * 16 + e] = inv4Elem(T[3], e);  // Camera::cameraMatrix: inverse of the absolute transform
                else T[2][e] = mul4Elem(T[1], T[7], e);
            }
            __syncwarp();
            if (half == 1) inst[L.slot_bars + i].model[e] = mul4Elem(T[2], T[4], e);  // r4
            if (lane >= 16 && lane < 28) {  // mesh / colour / segmentation tag / padding words of the three instances
                const int which = (lane - 16) >> 2, w = (lane - 16) & 3;
                const int agentColors[7] = {0, 1, 3, 7, 14, 10, 12};  // const.hpp:85 as palette indices
                MvInstance &d = inst[(which == 0 ? L.slot_eyes : (which == 1 ? L.slot_bars : L.slot_body)) + i];
                const int mesh = which == 2 ? 1 : 0, color = which == 0 ? 6 : (which == 1 ? 3 : agentColors[i % 7]);  // AGENT_EYES = DARK_NAVY, bar BLUE
                if (w == 0) d.mesh = mesh; else if (w == 1) d.color = color; else d.pad[w - 2] = w == 2 ? segTag(MV_SEG_AGENT, i) : 0;
            }
            __syncwarp();
        }
    }
    // reward diamonds: two cones each (layout_utils.cpp:114-126), rewritten only at reset and when one is collected
    const int nr = L.n_reward;
    for (int i = lane; i < nr; i += 32) {
        const bool alive = (S.env.reward_alive[i >> 5] >> (i & 31)) & 1u;
        if (!writeStatic && !((S.rewardDirty[i >> 5] >> (i & 31)) & 1u)) continue;
        M4 root = loadM4(L.reward_root[i]);
        if (!alive) {  // collected: moved away by 1000 (Obstacles :224, HexExplore :54), 500 (Collect :157) or 100 (HexMemory :108)
            const float far = L.scenario == MV_SCENARIO_COLLECT ? 500.0f : (L.scenario == MV_SCENARIO_HEX_MEMORY ? 100.0f : 1000.0f);
            root = mul4(translation4(v3(far, far, far)), root);
        }
        const int slot0 = L.reward_slot[i], mesh = L.reward_mesh[i], cnt = L.reward_cnt[i];
        putInstance(inst[slot0], root, mesh, L.reward_voxel[i][3], segTag(MV_SEG_REWARD, i));
        for (int k = 1; k < cnt; ++k)
            putInstance(inst[slot0 + k], mul4(root, mesh == 3 ? loadM4(L.cone_bottom_local) : loadM4(L.reward_child[i][k - 1])), mesh, L.reward_voxel[i][3],
                        segTag(MV_SEG_REWARD, i));
    }
    if (lane == 0) {
        counts[0] = L.mesh_counts[0]; counts[1] = L.mesh_counts[0] + L.mesh_counts[1] + L.mesh_counts[2] + L.mesh_counts[3] + L.mesh_counts[4];
        counts[2] = L.mesh_counts[1]; counts[3] = L.mesh_counts[2]; counts[4] = L.mesh_counts[3]; counts[5] = L.mesh_counts[4]; counts[6] = 0; counts[7] = 0;
    }
    (void)no;
}

// ---------------------------------------------------------------- state tensors (option "state_tensors")
// One env's rows, from the warp's state and the instance list `inst` that writeInstances has just written (its writes are visible to
// the warp after a __syncwarp).  An object's position is the translation column of its instance's model matrix, so a carried object is
// where it is drawn.  `all`: every object and reward row (an episode start, a terminal row); otherwise only the objects writeInstances
// rewrote (carried, or picked up / put down / pushed in this call) and the rewards collected in this call -- no other row can have changed.
__device__ float stateRewardValue(const WarpShared &S, const MvLevel &L, int i) {
    if (!((S.env.reward_alive[i >> 5] >> (i & 31)) & 1u)) return 0.0f;
    const bool penalty = L.scenario == MV_SCENARIO_COLLECT ? L.reward_voxel[i][3] != 1  // not GREEN
                                                          : (L.scenario == MV_SCENARIO_HEX_MEMORY && !((L.reward_good[i >> 5] >> (i & 31)) & 1u));
    return penalty ? -1.0f : 1.0f;
}
__device__ void writeStateRows(const WarpShared &S, const MvLevel &L, const MvInstance *inst, int A, bool all, float *ag, float *en, float *ob, float *rw, int lane) {
    for (int w = lane; w < A * 16; w += 32) {
        const MvAgent &a = S.agents[w >> 4];
        const int c = w & 15;
        float v;
        if (c < 3) v = a.pos[c];
        else if (c < 7) v = a.basis[c == 3 ? 0 : (c == 4 ? 2 : (c == 5 ? 6 : 8))];
        else if (c == 7) v = a.cur_x;
        else if (c < 11) v = a.hvel[c - 8];
        else if (c == 11) v = a.vvel;
        else if (c == 12) v = float(a.was_on_ground);
        else if (c == 13) v = float(a.was_jumping);
        else if (c == 14) v = float(a.carrying);
        else v = a.total_reward;
        ag[w] = v;
    }
    if (lane < 16) {
        const MvEnvState &e = S.env;
        const float v[11] = {e.episode_sec, L.episode_len, float(e.num_frames), float(L.scenario), float(L.n_obj), float(L.n_reward), float(e.solved),
                             float(e.reached_exit), float(e.highest_tower), e.bz_reward, float(e.positive_collected)};
        en[lane] = lane < 11 ? v[lane] : 0.0f;
    }
    auto objectRow = [&](int i, float *row) {
        const MvObject &o = S.objects[i];
        const float *m = inst[MV_OBJ_SLOT(o.meta)].model;
        row[0] = m[12]; row[1] = m[13]; row[2] = m[14]; row[3] = float(o.parent);
    };
    auto rewardRow = [&](int i, float *row) {
        row[0] = L.reward_root[i][12]; row[1] = L.reward_root[i][13]; row[2] = L.reward_root[i][14]; row[3] = stateRewardValue(S, L, i);
    };
    if (all) {
        for (int i = lane; i < MV_MAX_OBJECTS; i += 32) {
            float4 *row = reinterpret_cast<float4 *>(ob) + i;
            if (i < L.n_obj) { float r[4]; objectRow(i, r); *row = make_float4(r[0], r[1], r[2], r[3]); }
            else *row = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
        for (int i = lane; i < MV_MAX_REWARD; i += 32) {
            float4 *row = reinterpret_cast<float4 *>(rw) + i;
            if (i < L.n_reward) { float r[4]; rewardRow(i, r); *row = make_float4(r[0], r[1], r[2], r[3]); }
            else *row = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
        return;
    }
    for (int idx = lane; idx < A + S.nDirty; idx += 32) {
        const int i = idx < A ? S.agents[idx].carrying : S.objDirty[idx - A];
        if (i < 0) continue;
        float r[4]; objectRow(i, r);
        reinterpret_cast<float4 *>(ob)[i] = make_float4(r[0], r[1], r[2], r[3]);
    }
    for (int i = lane; i < L.n_reward; i += 32) {
        if (!((S.rewardDirty[i >> 5] >> (i & 31)) & 1u)) continue;
        float r[4]; rewardRow(i, r);
        reinterpret_cast<float4 *>(rw)[i] = make_float4(r[0], r[1], r[2], r[3]);
    }
}

// ---------------------------------------------------------------- the kernel
// kLevelSet: the level-set variant (StepParams::levelSet > 0).  A template parameter, not a run-time branch, so that the default
// variant is the code it was before level sets existed.  kState: the state-tensor variant (StepParams::stAgents set), kRC: the
// reward-component variant (StepParams::rcStep set, launched with kRcTickBytes more shared memory per warp), template parameters for the
// same reason.  kAuto: option "autoreset" (0 same-step, 1 next-step, 2 disabled; StepParams::awaiting set for 1 and 2).  Under 1 and 2
// an end does not flip: the env keeps the ended episode's scene in its live rows and is awaiting (MvEnvState::pad[1]) until the flip --
// its next active call under 1 (the forced-reset path, no tick), a restart under 2, where it is stepped as an inactive env meanwhile
template <bool kLevelSet, bool kState = false, bool kRC = false, int kAuto = 0> __global__ void __launch_bounds__(128) stepKernel(StepParams P) {
    extern __shared__ __align__(128) unsigned char smemRaw[];
    const int warpInBlock = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slotInGrid = blockIdx.x * (blockDim.x >> 5) + warpInBlock;
    // let the geometry kernel's blocks start right away: they synchronise per env on P.ready, not on this grid's completion
    asm volatile("griddepcontrol.launch_dependents;");
    if (slotInGrid >= P.E) return;
    const int env = P.envOrder ? int(__ldg(P.envOrder + slotInGrid)) : slotInGrid;
    const bool awaiting = kAuto != 0 && P.envs[env].pad[1] != 0;
    if ((P.active && !P.active[env]) || (kAuto == 2 && awaiting && !P.forceReset)) {
        // an inactive env: no staging, no tick, no write to its state.  It reports reward 0, not done and its unchanged true objective -- the
        // host mirror too, since a ring slot may still hold a value from three calls earlier -- and publishes its stamp for the raster launch
        for (int i = lane; i < P.A; i += 32) {
            const size_t idx = size_t(env) * P.A + i;
            P.rewards[idx] = 0.0f;
            if (P.hostRewards) { P.hostRewards[idx] = 0.0f; P.hostTrueObjectives[idx] = P.trueObjectives[idx]; }
        }
        if (kRC)  // step rows 0; the running and episode totals are left alone
            for (int i = lane; i < P.A * MV_R_COUNT; i += 32) P.rcStep[size_t(env) * P.A * MV_R_COUNT + i] = 0.0f;
        __syncwarp();
        if (lane == 0) {
            P.dones[env] = 0;
            P.doneReasons[env] = MV_END_NONE;
            if (P.hostDones) P.hostDones[env] = 0;
            if (P.hostDoneReasons) P.hostDoneReasons[env] = MV_END_NONE;
            if (kLevelSet && P.hostLevelIds) P.hostLevelIds[env] = P.levelIds[env];  // unchanged; the ring slot may hold an older call's
            if (kAuto) {
                P.awaiting[env] = awaiting;
                if (P.hostAwaiting) P.hostAwaiting[env] = awaiting;
            }
            __threadfence();
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(P.ready + env), "r"(P.readyStamp) : "memory");
        }
        return;
    }
    // a flip without physics: mv_reset / mv_reset_envs, or under next-step autoreset an awaiting env's active call.  An expression, not a
    // variable, so that under kAuto 0 every use reads P.forceReset as it did before the modes existed (and compiles to the same code)
#define MV_FORCED (P.forceReset || (kAuto == 1 && awaiting))
    WarpShared &S = reinterpret_cast<WarpShared *>(smemRaw)[warpInBlock];
    const int A = P.A;
    const float dt = P.k.dt;
    const long long tProf0 = P.prof ? clock64() : 0;
#define MV_PROBE(id) do { if (P.prof && lane == 0) P.prof[size_t(env) * 16 + (id)] = uint32_t(clock64() - tProf0); } while (0)

    // ---- stage state.  The movable-object records travel by one TMA bulk copy issued before anything else (its size is
    // the host-known bound on live object counts, so it does not wait for the env record); env + agents by plain loads.
    uint8_t *objGrid = P.objGrid + size_t(env) * P.gridCells;
    MvObject *gObjects = P.objects + size_t(env) * MV_MAX_OBJECTS;
    if (lane == 0) {
        mbarInit(&S.mbar, 1);
        if (!MV_FORCED) {
            const uint32_t bytes = uint32_t(P.maxObj) * uint32_t(sizeof(MvObject));
            mbarExpectTx(&S.mbar, bytes);
            if (bytes) bulkG2S(S.objects, gObjects, bytes, &S.mbar);
        }
    }
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(&P.envs[env]);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&S.env);
        for (int i = lane; i < int(sizeof(MvEnvState) / 4); i += 32) dst[i] = src[i];
        const uint32_t *asrc = reinterpret_cast<const uint32_t *>(&P.agents[size_t(env) * A]);
        uint32_t *adst = reinterpret_cast<uint32_t *>(&S.agents[0]);
        for (int i = lane; i < int(sizeof(MvAgent) / 4) * A; i += 32) adst[i] = asrc[i];
        if (lane == 0) { S.nDirty = 0; S.rewardDirty[0] = S.rewardDirty[1] = S.rewardDirty[2] = S.rewardDirty[3] = 0u; }
    }
    __syncwarp();
    int slot = S.env.slot;
    const MvLevel *L = &P.levels[levelRow<kLevelSet>(P, env, slot)];
    const MvBox *statics = P.statics + levelRow<kLevelSet>(P, env, slot) * size_t(P.staticCap);
    const float *staticRot = P.staticRot + levelRow<kLevelSet>(P, env, slot) * size_t(P.staticCap) * 2;
    int ns = L->n_static, no = L->n_obj;
    if (!MV_FORCED) mbarWait(&S.mbar, 0);

    bool resetNow = MV_FORCED;
    bool doneFlag = false;
    // lane i < A: agent i's reward summed over the call's ticks, in tick order from 0 (the tick that ends the episode pays 0, as one step does)
    float rewardSum = 0.0f;
    // kRC: this warp's tick columns, [agent][slot]; lane l folds entries l and l + 32 into rcCall by the rewardSum rule
    float *rcTick = kRC ? reinterpret_cast<float *>(smemRaw + sizeof(WarpShared) * (blockDim.x >> 5) + kRcTickBytes * warpInBlock) : nullptr;
    float rcCall[2] = {0.0f, 0.0f};
    MV_PROBE(0);  // state staged

    if (!MV_FORCED) {
        ColliderView cv;
        cv.S = &S; cv.L = L; cv.ns = ns; cv.no = no; cv.A = A; cv.nc = 0;

        // Action repeat: up to P.repeat ticks of the reference's step on the staged state, the same masks every tick except that Interact only
        // acts on tick 0 (it toggles carrying: one call is one press).  An episode end stops the ticks; what follows the loop (outputs, terminal
        // row, flip, write-back, instance list) sees the state of the tick that ended it, or of the last tick.
        for (int tick = 0; tick < P.repeat; ++tick) {
            for (int i = lane; i < MV_MAX_AGENTS; i += 32) S.lastReward[i] = 0.0f;
            if (kRC)
                for (int i = lane; i < MV_MAX_AGENTS * MV_R_COUNT; i += 32) rcTick[i] = 0.0f;
            if (lane == 0) S.memoryNear = 0u;
            __syncwarp();

            // ---- action phase (env.cpp:89-122)
            for (int i = 0; i < A; ++i) {
                MvAgent &a = S.agents[i];
                const int act = P.actions[size_t(env) * A + i];
                M3 basis;
                for (int k = 0; k < 9; ++k) basis.r[k] = a.basis[k];
                // forwardDirection / strafeLeftDirection use the basis BEFORE this step's look rotation? No: acceleration terms
                // are gathered first, then look is applied (env.cpp:95-113) -- same order here.
                V3 acc = v3(0, 0, 0);
                const V3 fwd = btNormalized(v3(basis.r[6], basis.r[7], -basis.r[8]));
                const V3 left = btNormalized(v3(-basis.r[0], basis.r[1], basis.r[2]));
                if (act & MV_A_FORWARD) acc = acc + fwd;
                else if (act & MV_A_BACKWARD) acc = acc - fwd;
                if (act & MV_A_LEFT) acc = acc + left;
                else if (act & MV_A_RIGHT) acc = acc - left;
                if (act & (MV_A_LOOKLEFT | MV_A_LOOKRIGHT)) {
                    M3 rot;
                    const float *src = (act & MV_A_LOOKLEFT) ? P.k.look_left : P.k.look_right;
                    for (int k = 0; k < 9; ++k) rot.r[k] = src[k];
                    basis = mul3(basis, rot);
                }
                float curX = a.cur_x;
                M4 cam = loadM4(a.cam_local);
                const float lim = L->look_limit;
                if (act & MV_A_LOOKUP) {
                    cam = mul4(cam, rotationX4(-curX));
                    curX += 1.5f * dt;
                    curX = lim < curX ? lim : curX;
                    cam = mul4(cam, rotationX4(curX));
                } else if (act & MV_A_LOOKDOWN) {
                    cam = mul4(cam, rotationX4(-curX));
                    curX -= 1.5f * dt * 1.1f;
                    curX = -lim < curX ? curX : -lim;
                    cam = mul4(cam, rotationX4(curX));
                }
                Kcc k;
                k.pos = v3(a.pos[0], a.pos[1], a.pos[2]); k.hvel = v3(a.hvel[0], a.hvel[1], a.hvel[2]);
                k.jumpAxis = v3(a.jump_axis[0], a.jump_axis[1], a.jump_axis[2]);
                k.vvel = a.vvel; k.voff = a.voff; k.stepOff = a.step_off; k.jumpSpeed = a.jump_speed;
                k.wasOnGround = a.was_on_ground != 0; k.wasJumping = a.was_jumping != 0;
                kccSetAcceleration(k, acc, dt);
                if ((act & MV_A_JUMP) && k.onGround()) {  // agent.cpp:157-161, KCC::jump :625-644
                    const V3 jv = v3(0, 6.2f, 0);
                    k.jumpSpeed = length(jv);
                    k.vvel = k.jumpSpeed;
                    k.wasJumping = true;
                    k.jumpAxis = btNormalized(jv);
                }
                __syncwarp();
                if (lane == 0) {
                    for (int q = 0; q < 9; ++q) a.basis[q] = basis.r[q];
                    a.cur_x = curX;
                    storeM4(a.cam_local, cam);
                    a.hvel[0] = k.hvel.x; a.hvel[1] = k.hvel.y; a.hvel[2] = k.hvel.z;
                    a.vvel = k.vvel; a.jump_speed = k.jumpSpeed; a.was_jumping = k.wasJumping;
                    a.jump_axis[0] = k.jumpAxis.x; a.jump_axis[1] = k.jumpAxis.y; a.jump_axis[2] = k.jumpAxis.z;
                }
                __syncwarp();
            }

            MV_PROBE(1);  // action phase
            // ---- stepSimulation: action interfaces in agent order (env.cpp:126)
            for (int i = 0; i < A; ++i) {
                MvAgent &a = S.agents[i];
                Kcc k;
                k.pos = v3(a.pos[0], a.pos[1], a.pos[2]); k.hvel = v3(a.hvel[0], a.hvel[1], a.hvel[2]);
                k.jumpAxis = v3(a.jump_axis[0], a.jump_axis[1], a.jump_axis[2]);
                k.vvel = a.vvel; k.voff = a.voff; k.stepOff = a.step_off; k.jumpSpeed = a.jump_speed;
                k.wasOnGround = a.was_on_ground != 0; k.wasJumping = a.was_jumping != 0;
                const V3 envLo = envelopeLo(k.pos), envHi = envelopeHi(k.pos);
                cv.nc = gatherCandidates(S, statics, staticRot, L->n_static_pre, ns, no, A, i, envLo, envHi, lane);
                if (i == 0) { MV_PROBE(2); if (P.prof && lane == 0) P.prof[size_t(env) * 16 + 12] = uint32_t(cv.nc); }  // candidate list of agent 0
                kccPlayerStep(k, cv, ns + no + i, dt, P.k.max_slope_cos, lane);
    #ifdef MV_KCC_COUNTERS
                if (i == 0 && P.prof && lane == 0) { P.prof[size_t(env) * 16 + 9] = k.dbg[0]; P.prof[size_t(env) * 16 + 10] = k.dbg[1]; P.prof[size_t(env) * 16 + 11] = k.dbg[2]; P.prof[size_t(env) * 16 + 13] = k.dbg[3]; }
    #endif
                if (leftEnvelope(envLo, envHi, k.pos)) S.env.faults |= MV_FAULT_ENVELOPE;
                __syncwarp();
                if (lane == 0) {
                    a.pos[0] = k.pos.x; a.pos[1] = k.pos.y; a.pos[2] = k.pos.z;
                    a.hvel[0] = k.hvel.x; a.hvel[1] = k.hvel.y; a.hvel[2] = k.hvel.z;
                    a.vvel = k.vvel; a.voff = k.voff; a.step_off = k.stepOff;
                    a.was_on_ground = k.wasOnGround; a.was_jumping = k.wasJumping;
                }
                __syncwarp();
            }
            MV_PROBE(3);  // character controllers
            // agent->updateTransform() (env.cpp:128-129)
            for (int i = lane; i < A; i += 32) {
                M4 ot;
                if (updateTransform(S.agents[i], ot)) storeM4(S.agents[i].object_t, ot);
                else S.env.faults |= MV_FAULT_NAN;
            }
            __syncwarp();

            MV_PROBE(4);  // updateTransform
            if (L->scenario == MV_SCENARIO_HEX_MEMORY) {
                // lanes look for collectables within the collect radius of some agent; the ordered (rare) bookkeeping stays on lane 0
                for (int i = 0; i < A; ++i) {
                    const MvAgent &a = S.agents[i];
                    bool near = false;
                    for (int r = lane; r < L->n_reward; r += 32) {
                        if (!((S.env.reward_alive[r >> 5] >> (r & 31)) & 1u)) continue;
                        const V3 dlt = v3(L->reward_root[r][12] - a.object_t[12], L->reward_root[r][13] - a.object_t[13], L->reward_root[r][14] - a.object_t[14]);
                        if (sqrtf(dlt.x * dlt.x + dlt.y * dlt.y + dlt.z * dlt.z) < 1.0f) near = true;
                    }
                    if (__ballot_sync(FULL, near) && lane == 0) S.memoryNear |= 1u << i;
                }
                __syncwarp();
            }
            // ---- scenario step: interact, fall detection, shaping rewards -- scalar work, lane 0
            if (lane == 0) {
                MvEnvState &e = S.env;
                const float *rt = P.rtable + size_t(env) * A * MV_R_COUNT;
                // every term paid is also added, with kRC, to the paying slot's tick column of the agent it is paid to
                auto pay = [&](int slotR, int ai, float v) {
                    S.lastReward[ai] += v;
                    if (kRC) rcTick[ai * MV_R_COUNT + slotR] += v;
                };
                auto rewardAgent = [&](int slotR, int ai, float mult) { pay(slotR, ai, rt[ai * MV_R_COUNT + slotR] * mult); };
                auto rewardTeam = [&](int slotR, int ai, float mult) {
                    rewardAgent(slotR, ai, mult * (1 - rt[ai * MV_R_COUNT + MV_R_TEAM_SPIRIT]));
                    for (int j = 0; j < A; ++j) pay(slotR, j, rt[j * MV_R_COUNT + slotR] * rt[j * MV_R_COUNT + MV_R_TEAM_SPIRIT] * mult / A);
                };
                const float carryingScale = 0.78f, carryingScaleInverse = 1.0f / carryingScale;
                // RearrangeScenario::checkDone / countMatchingObjects (scenario_rearrange.cpp:134-177)
                auto rearrangeCheckDone = [&](int agentIdx) {
                    const int matches = rearrangeCountMatches(S, *L);
                    if (matches > int(e.reached_exit)) { rewardTeam(MV_R_REARRANGE_ONE_MORE, agentIdx, 1); e.reached_exit = uint32_t(matches); }
                    if (matches >= L->n_arr && !e.solved) {
                        e.solved = 1;
                        rewardTeam(MV_R_REARRANGE_ALL, agentIdx, 1);
                        const float t = L->episode_len - 0.3f;  // doneWithTimer (scenario.hpp:114-117)
                        e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                    }
                };
                // objects picked up, put down or pushed, each listed once however often it is touched
                auto markDirty = [&](int oi) {
                    for (int d = 0; d < S.nDirty; ++d)
                        if (S.objDirty[d] == oi) return;
                    S.objDirty[S.nDirty++] = oi;
                };
                const bool interactTick = tick == 0;  // action repeat: Interact acts on the call's first tick only
                const bool hasStacking = L->scenario != MV_SCENARIO_SOKOBAN && L->scenario != MV_SCENARIO_HEX_EXPLORE && L->scenario != MV_SCENARIO_HEX_MEMORY && L->scenario != MV_SCENARIO_EMPTY;
                // the object in voxel (x, y, z), grid index g.  The reference's voxel map is unbounded, the dense grid is not: outside it
                // (g < 0: put down beyond the level's edge, sunk into the void, or above the head-room) the object is the resting one
                // whose translation floors to the voxel -- every resting object sits at its voxel + 0.5
                auto objAt = [&](int g, int x, int y, int z) {
                    if (g >= 0) return int(objGrid[g]);
                    for (int k = 0; k < L->n_obj; ++k) {
                        const MvObject &ob = S.objects[k];
                        if (ob.parent < 0 && int(floorf(ob.t[0])) == x && int(floorf(ob.t[1])) == y && int(floorf(ob.t[2])) == z) return k;
                    }
                    return int(MV_NO_OBJECT);
                };
                for (int i = 0; i < A && hasStacking && interactTick; ++i) {  // ObjectStackingComponent (Sokoban and the hex mazes have none)
                    if (!(P.actions[size_t(env) * A + i] & MV_A_INTERACT)) continue;
                    MvAgent &a = S.agents[i];
                    const M4 objT = loadM4(a.object_t), cam = loadM4(a.cam_local);
                    const M4 pickAbs = mul4(mul4(objT, cam), pickupLocal());
                    if (a.carrying >= 0) {
                        const int oi = a.carrying;
                        MvObject &o = S.objects[oi];
                        const M4 local = tsMatrix(v3(o.t[0], o.t[1], o.t[2]), v3(o.s[0], o.s[1], o.s[2]));
                        const V3 t = translationOf(mul4(pickAbs, local));
                        int vx, vy, vz;
                        toVoxel(t, vx, vy, vz);
                        const int gi = gridIndex(*L, vx, vy, vz);
                        bool collidesWithAgent = false;
                        for (int j = 0; j < A; ++j) {
                            if (j == i) continue;
                            int cx, cy, cz;
                            toVoxel(v3(S.agents[j].object_t[12], S.agents[j].object_t[13], S.agents[j].object_t[14]), cx, cy, cz);
                            if (cx == vx && cy == vy && cz == vz) { collidesWithAgent = true; break; }
                        }
                        const uint32_t *sol = P.solid + levelRow<kLevelSet>(P, env, slot) * 3 * P.gridWords;
                        auto solidAt = [&](int g) { return g >= 0 && ((sol[g >> 5] >> (g & 31)) & 1u); };
                        const bool empty = !solidAt(gi) && objAt(gi, vx, vy, vz) == MV_NO_OBJECT;
                        // canPlaceObject: TowerBuilding only inside the building zone, default true elsewhere
                        bool canPlace = true;
                        if (L->scenario == MV_SCENARIO_TOWER) canPlace = inBuildingZone(*L, vx, vz);
                        else if (L->scenario == MV_SCENARIO_REARRANGE)  // scenario_rearrange.cpp:128-132
                            canPlace = abs(vx - L->work_center[0]) <= 2 && abs(vz - L->work_center[2]) <= 2;
                        if (empty && !collidesWithAgent && canPlace) {
                            while (true) {
                                const int by = vy - 1;
                                if (by < -30) break;
                                const int gb = gridIndex(*L, vx, by, vz);
                                if (solidAt(gb) || objAt(gb, vx, by, vz) != MV_NO_OBJECT) break;
                                vy = by;
                            }
                            const int gp = gridIndex(*L, vx, vy, vz);
                            if (gp >= 0) objGrid[gp] = uint8_t(oi);  // outside the grid the object's own translation records it
                            const V3 sc = scalingOf(local);
                            o.parent = -1;
                            o.s[0] = sc.x * carryingScaleInverse; o.s[1] = sc.y * carryingScaleInverse; o.s[2] = sc.z * carryingScaleInverse;
                            o.t[0] = float(vx) + 0.5f; o.t[1] = float(vy) + 0.5f; o.t[2] = float(vz) + 0.5f;
                            syncPoseScene(o);
                            o.enabled = !o.enabled;
                            a.carrying = -1;
                            markDirty(oi);
                            if (L->scenario == MV_SCENARIO_TOWER) {  // placedObject (scenario_tower_building.cpp:206-214)
                                if (inBuildingZone(*L, vx, vz)) mvBzInsert(e, vx, vy, vz);
                                const float newReward = towerReward(e);
                                const float delta = newReward - e.bz_reward;
                                e.bz_reward = newReward;
                                rewardTeam(MV_R_TOWER_BUILDING, i, delta);
                                const int hgt = vy - L->bz_min[1] + 1;
                                e.highest_tower = e.highest_tower > hgt ? e.highest_tower : hgt;
                            } else if (L->scenario == MV_SCENARIO_REARRANGE) rearrangeCheckDone(i);  // placedObject
                        }
                    } else {
                        const V3 pickup = translationOf(pickAbs);
                        int vx, vy, vz;
                        vx = int(lroundf(floorf(pickup.x))); vy = int(lroundf(floorf(pickup.y))); vz = int(lroundf(floorf(pickup.z)));
                        int pickupHeight = 0;
                        while (pickupHeight <= 1) {
                            const int g = gridIndex(*L, vx, vy, vz), ga = gridIndex(*L, vx, vy + 1, vz);
                            const int here = objAt(g, vx, vy, vz);
                            const bool hasAbove = objAt(ga, vx, vy + 1, vz) != MV_NO_OBJECT;
                            if (here != MV_NO_OBJECT && !hasAbove) {
                                MvObject &o = S.objects[here];
                                o.enabled = !o.enabled;
                                const M4 local = tsMatrix(v3(o.t[0], o.t[1], o.t[2]), v3(o.s[0], o.s[1], o.s[2]));
                                const V3 sc = scalingOf(local);
                                o.s[0] = sc.x * carryingScale; o.s[1] = sc.y * carryingScale; o.s[2] = sc.z * carryingScale;
                                o.t[0] = 0.0f; o.t[1] = -0.3f; o.t[2] = 0.0f;
                                o.parent = i;
                                a.carrying = here;
                                if (g >= 0) objGrid[g] = MV_NO_OBJECT;
                                markDirty(here);
                                if (L->scenario == MV_SCENARIO_TOWER) {  // pickedObject (scenario_tower_building.cpp:216-225)
                                    if (inBuildingZone(*L, vx, vz)) mvBzErase(e, vx, vy, vz);
                                    if (!a.picked_up) { rewardAgent(MV_R_TOWER_PICKED_UP, i, 1); a.picked_up = 1; }
                                } else if (L->scenario == MV_SCENARIO_REARRANGE) rearrangeCheckDone(i);  // pickedObject
                                break;
                            } else vy += 1;
                            ++pickupHeight;
                        }
                    }
                }
                const uint32_t *planes = P.solid + levelRow<kLevelSet>(P, env, slot) * 3 * P.gridWords;
                auto planeBit = [&](int plane, int g) { return g >= 0 && ((planes[size_t(plane) * P.gridWords + (g >> 5)] >> (g & 31)) & 1u); };
                // FallDetectionComponent::resetAgent (component_fall_detection.hpp:44-56) -> KinematicCharacterController::warp
                auto resetAgent = [&](int i) {
                    MvAgent &a = S.agents[i];
                    V3 p = v3(L->init_pos[i][0], L->init_pos[i][1], L->init_pos[i][2]);
                    while (p.y < 1000) {
                        int x, y, z;
                        toVoxel(p, x, y, z);
                        if (!planeBit(0, gridIndex(*L, x, y, z))) break;
                        p.y += 1;
                    }
                    const float halfVoxel = 1.0f / 2;
                    a.pos[0] = p.x + halfVoxel; a.pos[1] = p.y + halfVoxel; a.pos[2] = p.z + halfVoxel;
                    for (int q = 0; q < 9; ++q) a.basis[q] = (q % 4 == 0) ? 1.0f : 0.0f;  // warp(): rotation reset to identity
                    a.hvel[0] = a.hvel[1] = a.hvel[2] = 0.0f;
                    a.vvel = 0;
                };
                const bool hasFallDetection = L->scenario == MV_SCENARIO_TOWER || L->scenario == MV_SCENARIO_OBSTACLES || L->scenario == MV_SCENARIO_COLLECT;
                for (int i = 0; i < A && hasFallDetection; ++i)  // FallDetectionComponent::step
                    if (S.agents[i].object_t[13] < -20) {
                        resetAgent(i);
                        if (L->scenario == MV_SCENARIO_COLLECT) rewardAgent(MV_R_COLLECT_BAD, i, 1);  // agentFell (scenario_collect.cpp:214-218)
                    }
                if (L->scenario == MV_SCENARIO_HEX_MEMORY) {
                    // HexMemoryScenario::step (scenario_hex_memory.cpp:79-119); positive_collected = goodObjectsCollected, n_positive = #good
                    if (e.positive_collected >= L->n_positive && !e.solved) {
                        e.solved = 1;
                        const float t = L->episode_len - 0.3f;  // doneWithTimer()
                        e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                    }
                    for (int i = 0; i < A; ++i) {
                        if (!((S.memoryNear >> i) & 1u)) continue;
                        const MvAgent &a = S.agents[i];
                        const V3 t = v3(a.object_t[12], a.object_t[13], a.object_t[14]);
                        int ax, ay, az;
                        toVoxel(t, ax, ay, az);
                        for (int dx = -1; dx <= 1; ++dx)
                            for (int dz = -1; dz <= 1; ++dz)
                                for (int r = 0; r < L->n_reward; ++r) {  // the voxel's object list, insertion order
                                    if (!((e.reward_alive[r >> 5] >> (r & 31)) & 1u)) continue;
                                    if (L->reward_voxel[r][0] != ax + dx || L->reward_voxel[r][1] != ay || L->reward_voxel[r][2] != az + dz) continue;
                                    const V3 dlt = v3(L->reward_root[r][12] - t.x, L->reward_root[r][13] - t.y, L->reward_root[r][14] - t.z);
                                    const float distance = sqrtf(dlt.x * dlt.x + dlt.y * dlt.y + dlt.z * dlt.z);
                                    if (distance < 1.0f) {
                                        const bool good = (L->reward_good[r >> 5] >> (r & 31)) & 1u;
                                        rewardTeam(good ? MV_R_MEMORY_GOOD : MV_R_MEMORY_BAD, i, 1);
                                        e.positive_collected += good ? 1 : 0;
                                        e.reward_alive[r >> 5] &= ~(1u << (r & 31));
                                        S.rewardDirty[r >> 5] |= 1u << (r & 31);
                                    }
                                }
                    }
                } else if (L->scenario == MV_SCENARIO_HEX_EXPLORE) {
                    // HexExploreScenario::step (scenario_hex_explore.cpp:42-58): first agent within 1.2 of the diamond's floor point
                    for (int i = 0; i < A; ++i) {
                        const MvAgent &a = S.agents[i];
                        const V3 dlt = v3(a.object_t[12] - L->goal[0], a.object_t[13] - L->goal[1], a.object_t[14] - L->goal[2]);
                        const float distance = sqrtf(dlt.x * dlt.x + dlt.y * dlt.y + dlt.z * dlt.z);
                        if (double(distance) < 1.2 && !e.solved) {
                            e.solved = 1;
                            const float t = L->episode_len - 0.3f;  // doneWithTimer()
                            e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                            rewardTeam(MV_R_EXPLORE_SOLVED, i, 1);
                            e.reward_alive[0] &= ~1u;  // rewardObject->translate({1e3, 1e3, 1e3})
                            S.rewardDirty[0] |= 1u;
                            break;
                        }
                    }
                } else if (L->scenario == MV_SCENARIO_SOKOBAN) {
                    // SokobanScenario::step (scenario_sokoban.cpp:168-222): push the box in front of the agent one cell further.  The grid
                    // has voxelSize 2; terrain plane 1 = SOKO_WALL, plane 2 = SOKO_GOAL
                    auto vox2 = [&](V3 p, int &x, int &y, int &z) { toVoxel(v3(p.x / 2.0f, p.y / 2.0f, p.z / 2.0f), x, y, z); };
                    for (int i = 0; i < A && interactTick; ++i) {
                        if (!(P.actions[size_t(env) * A + i] & MV_A_INTERACT)) continue;
                        const MvAgent &a = S.agents[i];
                        const M4 pickAbs = mul4(mul4(loadM4(a.object_t), loadM4(a.cam_local)), pickupLocal());
                        int bx, by, bz;
                        vox2(translationOf(pickAbs), bx, by, bz);
                        const int gb = gridIndex(*L, bx, by, bz);
                        if (gb < 0 || objGrid[gb] == MV_NO_OBJECT) continue;
                        int ax, ay, az;
                        vox2(v3(a.object_t[12], a.object_t[13], a.object_t[14]), ax, ay, az);
                        if (abs(ax - bx) + abs(ay - by) + abs(az - bz) != 1) continue;
                        const int dx = bx - ax, dy = by - ay, dz = bz - az;
                        const int tx = bx + dx, ty = by + dy, tz = bz + dz;
                        bool occupied = false;
                        for (int j = 0; j < A; ++j) {
                            int cx, cy, cz;
                            vox2(v3(S.agents[j].object_t[12], S.agents[j].object_t[13], S.agents[j].object_t[14]), cx, cy, cz);
                            if (cx == tx && cy == ty && cz == tz) { occupied = true; break; }
                        }
                        if (occupied) continue;
                        const int gt = gridIndex(*L, tx, ty, tz);
                        if (gt < 0) { e.faults |= MV_FAULT_GRID_RANGE; continue; }
                        if (planeBit(1, gt) || objGrid[gt] != MV_NO_OBJECT) continue;  // wall, or another box
                        const int oi = objGrid[gb];
                        MvObject &o = S.objects[oi];
                        objGrid[gt] = uint8_t(oi); objGrid[gb] = MV_NO_OBJECT;
                        // parent()->translate(delta * voxelSize): T(v) * (T(t) * S(s)) -- translation column = v*1 + t summed as the product does
                        const M4 moved = mul4(translation4(v3(float(dx) * 2.0f, float(dy) * 2.0f, float(dz) * 2.0f)), tsMatrix(v3(o.t[0], o.t[1], o.t[2]), v3(o.s[0], o.s[1], o.s[2])));
                        o.t[0] = moved.c[12]; o.t[1] = moved.c[13]; o.t[2] = moved.c[14];
                        syncPoseScene(o);
                        markDirty(oi);
                        const bool fromGoal = planeBit(2, gb), toGoal = planeBit(2, gt);
                        if (!fromGoal && toGoal) {
                            e.positive_collected += 1;
                            rewardTeam(MV_R_SOKOBAN_ON_TARGET, i, 1);
                            if (e.positive_collected == no && !e.solved) {
                                e.solved = 1;
                                rewardTeam(MV_R_SOKOBAN_ALL, i, 1);
                                const float t = L->episode_len - 0.3f;  // doneWithTimer()
                                e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                            }
                        } else if (fromGoal && !toGoal) {
                            e.positive_collected -= 1;
                            rewardTeam(MV_R_SOKOBAN_LEAVES_TARGET, i, 1);
                        }
                    }
                } else if (L->scenario == MV_SCENARIO_TOWER) {
                    // shaping: carrying an object inside the building zone (scenario_tower_building.cpp:184-198)
                    for (int i = 0; i < A; ++i) {
                        MvAgent &a = S.agents[i];
                        if (a.carrying >= 0) {
                            int x, y, z;
                            toVoxel(v3(a.object_t[12], a.object_t[13], a.object_t[14]), x, y, z);
                            if (inBuildingZone(*L, x, z) && !a.visited_bz) {
                                rewardTeam(MV_R_TOWER_VISITED_BZ, i, 1);
                                a.visited_bz = 1;
                            }
                        }
                    }
                } else if (L->scenario == MV_SCENARIO_COLLECT) {
                    // CollectScenario::step (scenario_collect.cpp:150-177)
                    for (int i = 0; i < A; ++i) {
                        MvAgent &a = S.agents[i];
                        int x, y, z;
                        toVoxel(v3(a.object_t[12], a.object_t[13], a.object_t[14]), x, y, z);
                        for (int r = 0; r < L->n_reward; ++r)
                            if (((e.reward_alive[r >> 5] >> (r & 31)) & 1u) && L->reward_voxel[r][0] == x && L->reward_voxel[r][1] == y && L->reward_voxel[r][2] == z) {
                                e.reward_alive[r >> 5] &= ~(1u << (r & 31));
                                S.rewardDirty[r >> 5] |= 1u << (r & 31);
                                const bool good = L->reward_voxel[r][3] == 1;  // GREEN palette index
                                if (good) { ++e.positive_collected; rewardTeam(MV_R_COLLECT_GOOD, i, 1); }
                                else rewardTeam(MV_R_COLLECT_BAD, i, 1);
                                if (e.positive_collected >= L->n_positive && !e.solved) {
                                    e.solved = 1;
                                    const float t = L->episode_len - 0.3f;  // doneWithTimer()
                                    e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                                    rewardTeam(MV_R_COLLECT_ALL, i, 1);
                                }
                                const int g = gridIndex(*L, x, y, z);  // vg.grid.remove(voxel): the whole entry goes, incl. an object parked in it
                                if (g >= 0) objGrid[g] = MV_NO_OBJECT;
                            }
                    }
                } else if (L->scenario == MV_SCENARIO_OBSTACLES) {
                    // ObstaclesScenario::step (scenario_obstacles.cpp:202-238)
                    int numAgentsAtExit = 0;
                    for (int i = 0; i < A; ++i) {
                        MvAgent &a = S.agents[i];
                        int x, y, z;
                        toVoxel(v3(a.object_t[12], a.object_t[13], a.object_t[14]), x, y, z);
                        const int g = gridIndex(*L, x, y, z);
                        if (planeBit(1, g)) {
                            ++numAgentsAtExit;
                            if (!((e.reached_exit >> i) & 1u)) {
                                e.reached_exit |= 1u << i;
                                rewardTeam(MV_R_OBST_AGENT_AT_EXIT, i, 1);
                                if (a.carrying >= 0) rewardTeam(MV_R_OBST_CARRIED_TO_EXIT, i, 1);
                            }
                        } else if (planeBit(2, g))
                            resetAgent(i);  // agentTouchedLava
                        for (int r = 0; r < L->n_reward; ++r)
                            if (((e.reward_alive[r >> 5] >> (r & 31)) & 1u) && L->reward_voxel[r][0] == x && L->reward_voxel[r][1] == y && L->reward_voxel[r][2] == z) {
                                e.reward_alive[r >> 5] &= ~(1u << (r & 31));
                                S.rewardDirty[r >> 5] |= 1u << (r & 31);
                                rewardTeam(MV_R_OBST_EXTRA, i, 1);
                            }
                    }
                    if (numAgentsAtExit == A && !e.solved) {
                        e.solved = 1;
                        const float t = L->episode_len - 0.3f;  // doneWithTimer() (scenario.hpp:114-117)
                        e.episode_sec = e.episode_sec > t ? e.episode_sec : t;
                        for (int i = 0; i < A; ++i) rewardAgent(MV_R_OBST_ALL_AT_EXIT, i, 1);  // rewardAll
                    }
                }
                // env.cpp:133-152
                e.episode_sec += dt;
                const float len = L->episode_len;
                {
                    const float frac0 = (len - e.episode_sec) / len;
                    const float frac = frac0 > 0.0f ? frac0 : 0.0f;
                    for (int i = 0; i < A; ++i) {
                        MvAgent &a = S.agents[i];
                        const float req[3] = {frac * 0.24f, float(0.0015), float(0.001)};
                        for (int q = 0; q < 3; ++q) {
                            const float sc = sqrtf(a.bar_scale[q] * a.bar_scale[q] + 0.0f * 0.0f + 0.0f * 0.0f);
                            a.bar_scale[q] = a.bar_scale[q] * (req[q] / sc);
                        }
                    }
                }
                for (int i = 0; i < A; ++i) S.agents[i].total_reward += S.lastReward[i];
                e.num_frames += 1;
                // a requested end (mv_step_device_ends) is a timer end after the call's last tick; with two level slots, before the episode's
                // third call the env's next level may not be staged yet (every call of an episode but one that ends runs all its ticks, so that
                // is 3 * repeat ticks).  Four slots always hold the next level, and so does a level set
                const bool requested = P.ends && P.ends[env] && tick == P.repeat - 1 && (kLevelSet || P.slots != 2 || e.num_frames >= 3 * P.repeat);
                S.doneFlag = (e.episode_sec >= len || requested) ? 1 : 0;
            }
            __syncwarp();
            doneFlag = S.doneFlag != 0;
            if (doneFlag) break;
            if (lane < A) rewardSum += S.lastReward[lane];
            if (kRC) { rcCall[0] += rcTick[lane]; rcCall[1] += rcTick[lane + 32]; }
        }
        // same-step autoreset flips at the end; the other modes keep the ended episode live and mark the env awaiting its flip
        resetNow = kAuto == 0 && doneFlag;
        if (kAuto && doneFlag && lane == 0) S.env.pad[1] = 1;
        MV_PROBE(5);  // scenario logic
    }

    // ---- outputs of the finished step; VectorEnv::step captures trueObjective BEFORE reset and the rewards AFTER it (zeroed)
    // Host mirrors (pinned, mapped) are written by the kernel itself when given: no copy operations between the kernels
    // of successive steps.
    for (int i = lane; i < A; i += 32) {
        const size_t idx = size_t(env) * A + i;
        float to = P.trueObjectives[idx];
        if (!MV_FORCED && doneFlag) { to = L->scenario == MV_SCENARIO_TOWER ? float(S.env.highest_tower) : float(S.env.solved); P.trueObjectives[idx] = to; }
        const float r = MV_FORCED ? 0.0f : rewardSum;  // i == lane: A <= MV_MAX_AGENTS < 32
        P.rewards[idx] = r;
        if (P.hostRewards) { P.hostRewards[idx] = r; P.hostTrueObjectives[idx] = to; }
    }
    if (kRC) {  // the step rows; the running totals take them in call order, and an end moves its total to the episode rows
        const size_t base = size_t(env) * A * MV_R_COUNT;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int i = lane + 32 * k;
            if (i < A * MV_R_COUNT) {
                const float s = MV_FORCED ? 0.0f : rcCall[k];
                P.rcStep[base + i] = s;
                if (MV_FORCED) {
                    P.rcRun[base + i] = 0.0f;
                } else if (doneFlag) {
                    P.rcEpisode[base + i] = P.rcRun[base + i] + s;
                    P.rcRun[base + i] = 0.0f;
                } else {
                    P.rcRun[base + i] += s;
                }
            }
        }
    }
    if (lane == 0) {
        const uint8_t dn = (!MV_FORCED && doneFlag) ? 1 : 0;
        P.dones[env] = dn;
        if (P.hostDones) P.hostDones[env] = dn;
        // solved first: doneWithTimer ran (also when a request arrives during its grace), then the clock, else the caller's request
        const uint8_t why = !dn ? uint8_t(MV_END_NONE) : (S.env.solved ? uint8_t(MV_END_SOLVED) : (S.env.episode_sec >= L->episode_len ? uint8_t(MV_END_TIME) : uint8_t(MV_END_REQUESTED)));
        P.doneReasons[env] = why;
        if (P.hostDoneReasons) P.hostDoneReasons[env] = why;
        if (kAuto) {  // an env that ends awaits its flip; one that ran no tick flips below (or was not awaiting)
            P.awaiting[env] = dn;
            if (P.hostAwaiting) P.hostAwaiting[env] = dn;
        }
    }

    if (kAuto == 0 && P.termInstances && !MV_FORCED && doneFlag) {
        // terminal row: the live row as the previous step left it, with this step's dynamic entries written on top from the still-live
        // level slot.  writeInstances only reads S, so this is exactly what a step that does not end writes, and the live path below
        // is untouched.
        MvInstance *tInst = P.termInstances + size_t(env) * P.instStride;
        int32_t *tCounts = P.termCounts + size_t(env) * 8;
        float *tViews = P.termViews + size_t(env) * A * 16;
        const int32_t *counts = P.instCounts + size_t(env) * 8;
        const uint32_t *src = reinterpret_cast<const uint32_t *>(P.instances + size_t(env) * P.instStride);
        uint32_t *dst = reinterpret_cast<uint32_t *>(tInst);
        const int words = counts[1] * int(sizeof(MvInstance) / 4);
        for (int i = lane; i < words; i += 32) dst[i] = src[i];
        if (lane < 8) tCounts[lane] = counts[lane];
        for (int i = lane; i < A * 16; i += 32) tViews[i] = P.views[size_t(env) * A * 16 + i];
        __syncwarp();
        writeInstances(S, *L, statics, P.deco + levelRow<kLevelSet>(P, env, slot) * P.decoCap, tInst, tCounts, tViews, A, /*writeStatic=*/false, lane);
        __syncwarp();
        if (kState && P.termStAgents) {  // the state this terminal frame shows: after the ending tick, before the flip
            writeStateRows(S, *L, tInst, A, /*all=*/true, P.termStAgents + size_t(env) * A * 16, P.termStEnvs + size_t(env) * 16,
                           P.termStObjects + size_t(env) * MV_MAX_OBJECTS * 4, P.termStRewards + size_t(env) * MV_MAX_REWARD * 4, lane);
            __syncwarp();
        }
    }

    if (resetNow) {
        if (kAuto && lane == 0) S.env.pad[1] = 0;
        if (kLevelSet) {
            // level set: the next level is a row of the bank, chosen here -- the caller's choice when it names a level of the set (used once),
            // else the hash of the env's pick seed and the new episode's index.  The entry comes from outside the engine: it is bounded
            // before it indexes anything, and a value out of range is left alone and ignored.  Bank rows are always there: no serial check.
            // A row being replaced is not pickable: an entry naming it stays for a later end, and the hash probes forward to the next row
            if (lane == 0) {
                S.env.episode_idx += 1;
                const int base = P.bankBase[env];
                int j = P.nextLevels[env];
                if (j >= 0 && j < P.levelSet && P.rowPickable[base + j]) {
                    P.nextLevels[env] = -1;
                } else {
                    j = int(mvLevelSetPick(uint32_t(S.env.pad[0]), S.env.episode_idx, P.levelSet));
                    for (int k = 0; k < P.levelSet && !P.rowPickable[base + j]; ++k) j = j + 1 == P.levelSet ? 0 : j + 1;
                }
                S.env.slot = base + j;
            }
            __syncwarp();
            slot = S.env.slot;
        } else {
            // flip to the pre-staged next level (episode end, or mv_reset forcing a new episode everywhere): the slots form a ring
            slot = slot + 1 == P.slots ? 0 : slot + 1;
        }
        L = &P.levels[levelRow<kLevelSet>(P, env, slot)];
        statics = P.statics + levelRow<kLevelSet>(P, env, slot) * size_t(P.staticCap);
        staticRot = P.staticRot + levelRow<kLevelSet>(P, env, slot) * size_t(P.staticCap) * 2;
        if (lane == 0 && !kLevelSet) {
            S.env.slot = slot;
            S.env.episode_idx += 1;
            if (L->serial != S.env.episode_idx) S.env.faults |= MV_FAULT_LEVEL_NOT_READY;
        }
        __syncwarp();
        ns = L->n_static; no = L->n_obj;
        resetEnv(S, *L, objGrid, A, lane);
        // all objects are fresh: write the whole array back
        {
            const uint32_t *src = reinterpret_cast<const uint32_t *>(&S.objects[0]);
            uint32_t *dst = reinterpret_cast<uint32_t *>(gObjects);
            for (int i = lane; i < int(sizeof(MvObject) / 4) * no; i += 32) dst[i] = src[i];
        }
    } else {
        // write back the (at most 2A) objects touched this step
        const int nd = S.nDirty;
        for (int d = 0; d < nd; ++d) {
            const int oi = S.objDirty[d];
            const uint32_t *src = reinterpret_cast<const uint32_t *>(&S.objects[oi]);
            uint32_t *dst = reinterpret_cast<uint32_t *>(&gObjects[oi]);
            for (int i = lane; i < int(sizeof(MvObject) / 4); i += 32) dst[i] = src[i];
        }
    }
    __syncwarp();
    MV_PROBE(6);  // outputs, flip/reset, object write-back

    writeInstances(S, *L, statics, P.deco + levelRow<kLevelSet>(P, env, slot) * P.decoCap, P.instances + size_t(env) * P.instStride, P.instCounts + size_t(env) * 8, P.views + size_t(env) * A * 16, A, resetNow, lane);

    MV_PROBE(7);  // instance list + views
    if (kState) {  // the rows of the state the returned frame shows: after an end, the new episode's first
        __syncwarp();
        writeStateRows(S, *L, P.instances + size_t(env) * P.instStride, A, resetNow || (kAuto != 0 && doneFlag), P.stAgents + size_t(env) * A * 16, P.stEnvs + size_t(env) * 16,
                       P.stObjects + size_t(env) * MV_MAX_OBJECTS * 4, P.stRewards + size_t(env) * MV_MAX_REWARD * 4, lane);
    }

    // ---- commit env + agents
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(&S.env);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&P.envs[env]);
        for (int i = lane; i < int(sizeof(MvEnvState) / 4); i += 32) dst[i] = src[i];
        const uint32_t *asrc = reinterpret_cast<const uint32_t *>(&S.agents[0]);
        uint32_t *adst = reinterpret_cast<uint32_t *>(&P.agents[size_t(env) * A]);
        for (int i = lane; i < int(sizeof(MvAgent) / 4) * A; i += 32) adst[i] = asrc[i];
    }
    if (lane == 0 && S.env.faults && P.hostFaults) atomicOr_system(P.hostFaults, S.env.faults);  // sticky, rare
    MV_PROBE(8);  // commit
    // publish: everything this warp wrote (state, instance list, views, zeroed triangle counters) before the stamp
    __syncwarp();
    if (lane == 0) {
        if (kLevelSet) {  // the level the returned frame shows: after an end, the new episode's
            const int32_t id = S.env.slot - P.bankBase[env];
            P.levelIds[env] = id;
            if (P.hostLevelIds) P.hostLevelIds[env] = id;
        }
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(P.ready + env), "r"(P.readyStamp) : "memory");
    }
#undef MV_FORCED
#undef MV_PROBE
}

// ---------------------------------------------------------------- mv_debug_kcc: chosen contact cases through the step's own collision code
// One warp per case: the candidate gather, warpSweep / warpRecover / kccPlayerStep exactly as stepKernel runs them, on a caller-built
// collider set.  Layouts are those of mv_debug_kcc (include/megaverse_b200.h); the host entry validates them.
struct KccCaseParams {
    const int32_t *hdr;      // [n][8] n_static_pre, n_static, n_obj, A, mode, agent
    const MvBox *statics;    // [n][MV_MAX_OBJECTS]
    const float *staticRot;  // [n][MV_MAX_OBJECTS][2]
    const MvObject *objects; // [n][MV_MAX_OBJECTS] col_c, col_h, enabled
    const float *agentPos;   // [n][MV_MAX_AGENTS][3] (the querying agent's own is its position for the envelope)
    const float *query;      // [n][20]
    int32_t *outI;           // [n][8]
    float *outF;             // [n][16]
};
constexpr int kKccSweep = 0, kKccRecover = 1, kKccStep = 2;

__global__ void __launch_bounds__(32) kccCaseKernel(KccCaseParams P) {
    extern __shared__ __align__(128) unsigned char smemRaw[];
    WarpShared &S = *reinterpret_cast<WarpShared *>(smemRaw);
    __shared__ int16_t slotCollider[MV_MAX_CAND];
    const int cs = blockIdx.x, lane = threadIdx.x;
    const int32_t *hd = P.hdr + size_t(cs) * 8;
    const int nsPre = hd[0], ns = hd[1], no = hd[2], A = hd[3], mode = hd[4], i = hd[5];
    const float *q = P.query + size_t(cs) * 20;
    for (int o = lane; o < no; o += 32) S.objects[o] = P.objects[size_t(cs) * MV_MAX_OBJECTS + o];
    for (int a = lane; a < A; a += 32)
        for (int c = 0; c < 3; ++c) S.agents[a].pos[c] = (mode == kKccStep && a == i) ? q[c] : P.agentPos[(size_t(cs) * MV_MAX_AGENTS + a) * 3 + c];
    if (lane == 0) S.env.faults = 0;
    __syncwarp();
    const V3 self = v3(S.agents[i].pos[0], S.agents[i].pos[1], S.agents[i].pos[2]);
    const V3 envLo = envelopeLo(self), envHi = envelopeHi(self);
    ColliderView cv;
    cv.S = &S; cv.L = nullptr; cv.ns = ns; cv.no = no; cv.A = A;
    cv.nc = gatherCandidates(S, P.statics + size_t(cs) * MV_MAX_OBJECTS, P.staticRot + size_t(cs) * MV_MAX_OBJECTS * 2, nsPre, ns, no, A, i, envLo, envHi,
                             lane, slotCollider);
    int32_t oi[8] = {cv.nc, 0, 0, -1, -1, 0, 0, 0};
    float of[16] = {};
    if (mode == kKccSweep) {
        const SweepReport r = warpSweep<true>(cv, ns + no + i, v3(q[0], q[1], q[2]), v3(q[3], q[4], q[5]), v3(q[6], q[7], q[8]), q[9], lane);
        oi[2] = r.hit;
        if (r.hit) { oi[3] = slotCollider[r.slot]; oi[4] = r.feature; }
        of[0] = r.fraction; of[1] = r.normal.x; of[2] = r.normal.y; of[3] = r.normal.z;
    } else if (mode == kKccRecover) {
        V3 delta = v3(0, 0, 0);
        int slot = -1;
        oi[2] = warpRecover<true>(cv, ns + no + i, v3(q[0], q[1], q[2]), delta, lane, &slot);
        if (oi[2]) { oi[3] = slotCollider[slot]; of[0] = delta.x; of[1] = delta.y; of[2] = delta.z; }
    } else {
        Kcc k;
        k.pos = v3(q[0], q[1], q[2]); k.hvel = v3(q[3], q[4], q[5]);
        k.vvel = q[6]; k.voff = q[7]; k.stepOff = q[8]; k.jumpSpeed = q[9];
        k.jumpAxis = v3(q[10], q[11], q[12]);
        k.wasOnGround = q[13] != 0.0f; k.wasJumping = q[14] != 0.0f;
        kccPlayerStep(k, cv, ns + no + i, q[15], q[16], lane);
        if (leftEnvelope(envLo, envHi, k.pos)) S.env.faults |= MV_FAULT_ENVELOPE;
        oi[2] = k.wasOnGround; oi[5] = k.wasJumping;
        of[0] = k.pos.x; of[1] = k.pos.y; of[2] = k.pos.z; of[3] = k.hvel.x; of[4] = k.hvel.y; of[5] = k.hvel.z;
        of[6] = k.vvel; of[7] = k.voff; of[8] = k.stepOff; of[9] = k.jumpSpeed;
    }
    __syncwarp();
    oi[1] = S.env.faults;
    if (lane < 8) P.outI[size_t(cs) * 8 + lane] = oi[lane];
    if (lane < 16) P.outF[size_t(cs) * 16 + lane] = of[lane];
}

}  // namespace mvk
