// ORACLE (test infrastructure, NOT product code): C entry points of the CPU restatement, loaded with ctypes by
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs ONLY.
// Mirrors MegaverseGym (src/libs/bindings/megaverse.cpp:36-243) + VectorEnv (src/libs/env/src/vector_env.cpp:89-120).
#include <array>
#include <atomic>
#include <thread>

#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "orc_raster.hpp"
#include "orc_maze.hpp"

using namespace orc;

// minimal parallel-for over envs (libgomp is not available in this image)
template <typename F> static void parallelFor(int n, int threads, F &&f) {
    if (threads <= 1 || n <= 1) { for (int i = 0; i < n; ++i) f(i); return; }
    std::atomic<int> next{0};
    auto worker = [&]() { for (int i = next++; i < n; i = next++) f(i); };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(worker);
    worker();
    for (auto &t : pool) t.join();
}

struct OrcVec {
    std::vector<std::unique_ptr<Env>> envs;
    int w, h, numEnvs, numAgents;
    std::vector<uint8_t> obs;
    std::vector<float> depth;
    std::vector<float> rewards, trueObjectives;
    std::vector<uint8_t> dones;
    Rng rng{std::random_device{}()};
    bool renderEnabled = true;
    bool wantDepth = false;
    int threads = 1;
    std::string error;

    void renderEnv(int e) {
        Env &env = *envs[size_t(e)];
        const auto inst = env.instances();
        for (int a = 0; a < numAgents; ++a) {
            const size_t view = size_t(e) * numAgents + a;
            renderView(env.viewMatrix(a), inst, w, h, obs.data() + view * size_t(w) * h * 4, wantDepth ? depth.data() + view * size_t(w) * h : nullptr);
        }
    }
};

extern "C" {

void *orc_create(const char *scenario, int w, int h, int numEnvs, int numAgents, const char **keys, const float *vals, int nparams) {
    auto *v = new OrcVec;
    try {
        FloatParams fp;
        for (int i = 0; i < nparams; ++i) fp[keys[i]] = vals[i];
        for (int i = 0; i < numEnvs; ++i) v->envs.emplace_back(std::make_unique<Env>(scenario, numAgents, fp));
    } catch (const std::exception &) {
        delete v;
        return nullptr;
    }
    v->w = w; v->h = h; v->numEnvs = numEnvs; v->numAgents = numAgents;
    const size_t N = size_t(numEnvs) * numAgents;
    v->obs.assign(N * w * h * 4, 0);
    v->depth.assign(N * w * h, 0.0f);
    v->rewards.assign(N, 0.0f);
    v->trueObjectives.assign(N, 0.0f);
    v->dones.assign(size_t(numEnvs), 0);
    return v;
}
void orc_destroy(void *p) { delete static_cast<OrcVec *>(p); }
void orc_set_options(void *p, int render, int depth, int threads) {
    auto *v = static_cast<OrcVec *>(p);
    v->renderEnabled = render != 0; v->wantDepth = depth != 0; v->threads = threads < 1 ? 1 : threads;
}
// MegaverseGym::seed (megaverse.cpp:60-69)
void orc_seed(void *p, int seedValue) {
    auto *v = static_cast<OrcVec *>(p);
    v->rng.seed((unsigned long)seedValue);
    for (auto &e : v->envs) e->seed(randRange(0, 1 << 30, v->rng));
}
// megaverse_test_app.cpp:250-254 seeds env i with 42+i directly
void orc_seed_env(void *p, int env, int seedValue) { static_cast<OrcVec *>(p)->envs[size_t(env)]->seed(seedValue); }

// VectorEnv::reset (vector_env.cpp:110-120)
void orc_reset(void *p) {
    auto *v = static_cast<OrcVec *>(p);
    parallelFor(v->numEnvs, v->threads, [&](int e) {
        v->envs[size_t(e)]->reset();
        if (v->renderEnabled) v->renderEnv(e);
    });
    std::fill(v->rewards.begin(), v->rewards.end(), 0.0f);
    std::fill(v->dones.begin(), v->dones.end(), 0);
}
void orc_set_actions(void *p, const int32_t *masks) {
    auto *v = static_cast<OrcVec *>(p);
    for (int e = 0; e < v->numEnvs; ++e)
        for (int a = 0; a < v->numAgents; ++a) v->envs[size_t(e)]->setAction(a, masks[e * v->numAgents + a]);
}
// VectorEnv::step (vector_env.cpp:89-108) + getLastRewards (megaverse.cpp:128-137)
void orc_step(void *p) {
    auto *v = static_cast<OrcVec *>(p);
    parallelFor(v->numEnvs, v->threads, [&](int e) {
        Env &env = *v->envs[size_t(e)];
        env.step();
        if (env.done) {
            v->dones[size_t(e)] = 1;
            for (int a = 0; a < v->numAgents; ++a) v->trueObjectives[size_t(e) * v->numAgents + a] = env.trueObjective(a);
            env.reset();
        } else {
            v->dones[size_t(e)] = 0;
        }
        for (int a = 0; a < v->numAgents; ++a) v->rewards[size_t(e) * v->numAgents + a] = env.lastReward[size_t(a)];
        if (v->renderEnabled) v->renderEnv(e);
    });
}
const uint8_t *orc_obs(void *p) { return static_cast<OrcVec *>(p)->obs.data(); }
const float *orc_depth(void *p) { return static_cast<OrcVec *>(p)->depth.data(); }
const float *orc_rewards(void *p) { return static_cast<OrcVec *>(p)->rewards.data(); }
const uint8_t *orc_dones(void *p) { return static_cast<OrcVec *>(p)->dones.data(); }
const float *orc_true_objectives(void *p) { return static_cast<OrcVec *>(p)->trueObjectives.data(); }
void orc_render_now(void *p) {
    auto *v = static_cast<OrcVec *>(p);
    parallelFor(v->numEnvs, v->threads, [&](int e) { v->renderEnv(e); });
}

int orc_get_reward_shaping(void *p, int env, int agent, const char *key, float *out) {
    auto &rs = static_cast<OrcVec *>(p)->envs[size_t(env)]->rewardShaping[size_t(agent)];
    auto it = rs.find(key);
    if (it == rs.end()) return 1;
    *out = it->second;
    return 0;
}
void orc_set_reward_shaping(void *p, int env, int agent, const char *key, float val) {
    static_cast<OrcVec *>(p)->envs[size_t(env)]->rewardShaping[size_t(agent)][key] = val;
}

// ---- introspection for parity tests -------------------------------------------------------------------------------
// level: ints.  [0]=numStaticBoxes [1]=numTerrain [2]=numObjects [3..8]=buildingZone min/max, then per static box 8 ints
// (min3,max3(inclusive),type,color), per terrain slab 7 ints (terrain,min3,max3), per object 3 ints (spawn voxel),
// then per agent 3 ints (spawn voxel)
int orc_get_level(void *p, int envIdx, int32_t *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(envIdx)];
    std::vector<int32_t> o;
    o.push_back(int(env.staticBoxes.size()));
    o.push_back(int(env.terrainSlabs.size()));
    o.push_back(int(env.objectSpawnPositions.size()));
    const BoundingBox bz = env.scenario == Env::S_TOWER ? env.buildingZone : BoundingBox{};
    for (int x : {bz.min.x, bz.min.y, bz.min.z, bz.max.x, bz.max.y, bz.max.z}) o.push_back(x);
    for (auto &sb : env.staticBoxes)
        for (int x : {sb.bb.min.x, sb.bb.min.y, sb.bb.min.z, sb.bb.max.x, sb.bb.max.y, sb.bb.max.z, int(sb.type), int(sb.color)}) o.push_back(x);
    for (auto &ts : env.terrainSlabs)
        for (int x : {ts.terrain, ts.bb.min.x, ts.bb.min.y, ts.bb.min.z, ts.bb.max.x, ts.bb.max.y, ts.bb.max.z}) o.push_back(x);
    for (auto &c : env.objectSpawnPositions)
        for (int x : {c.x, c.y, c.z}) o.push_back(x);
    for (auto &c : env.agentSpawnPositions)
        for (int x : {int(c.x), int(c.y), int(c.z)}) o.push_back(x);
    if (env.scenario != Env::S_TOWER) {  // scenario extras: numPlatforms, reward-object voxels
        o.push_back(env.scenario == Env::S_OBSTACLES ? env.numPlatforms : 0);
        o.push_back(int(env.rewardSpawnPositions.size()));
        for (auto &c : env.rewardSpawnPositions)
            for (int x : {c.x, c.y, c.z}) o.push_back(x);
        if (env.scenario == Env::S_HEX_EXPLORE || env.scenario == Env::S_HEX_MEMORY || env.scenario == Env::S_EMPTY) {  // free-standing colliders (bit patterns)
            o.push_back(env.agentColliderBase);
            for (int i = 0; i < env.agentColliderBase; ++i) {
                const Collider &c = env.colliders[size_t(i)];
                const float f[8] = {c.c.x, c.c.y, c.c.z, c.h.x, c.h.y, c.h.z, c.rotated ? c.ax : 1.0f, c.rotated ? c.az : 0.0f};
                int32_t w[8];
                std::memcpy(w, f, 32);
                for (int k = 0; k < 8; ++k) o.push_back(w[k]);
            }
        }
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::memcpy(out, o.data(), o.size() * sizeof(int32_t));
    return int(o.size());
}

// state: floats.  header 8: currEpisodeSec, episodeLengthSec, numFrames, highestTower, currBuildingZoneReward, numObjects,
// numColliders, done.  Per agent 28: pos3, basis9(row major), hvel3, vVel, vOffset, currentStepOffset, wasOnGround,
// wasJumping, jumpSpeed, currXRotation, carrying, totalReward, lastReward, pad.  Per object 9: translation3 (abs),
// scale3 (local), parentAgent, colliderEnabled, pad
int orc_get_state(void *p, int envIdx, float *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(envIdx)];
    std::vector<float> o;
    o.push_back(env.currEpisodeSec); o.push_back(env.episodeLengthSec()); o.push_back(float(env.numFrames)); o.push_back(float(env.highestTower));
    o.push_back(env.currBuildingZoneReward); o.push_back(float(env.objects.size())); o.push_back(float(env.colliders.size())); o.push_back(env.done ? 1.f : 0.f);
    for (int i = 0; i < env.numAgents; ++i) {
        const Agent &a = env.agents[size_t(i)];
        const KCC &k = a.kcc;
        for (float x : {k.pos.x, k.pos.y, k.pos.z}) o.push_back(x);
        for (int r = 0; r < 3; ++r) for (float x : {k.basis.r[r].x, k.basis.r[r].y, k.basis.r[r].z}) o.push_back(x);
        for (float x : {k.horizontalVelocity.x, k.horizontalVelocity.y, k.horizontalVelocity.z, k.verticalVelocity, k.verticalOffset, k.currentStepOffset,
                        k.wasOnGround ? 1.f : 0.f, k.wasJumping ? 1.f : 0.f, k.jumpSpeed, a.currXRotation, float(env.carryingObject[size_t(i)]),
                        env.totalReward[size_t(i)], env.lastReward[size_t(i)], 0.f})
            o.push_back(x);
    }
    for (int i = 0; i < int(env.objects.size()); ++i) {
        const MovableObject &ob = env.objects[size_t(i)];
        const Vec3 t = translationOf(env.objectAbs(i));
        for (float x : {t.x, t.y, t.z, ob.local.c[0][0], ob.local.c[1][1], ob.local.c[2][2], float(ob.parentAgent),
                        env.colliders[size_t(ob.collider)].enabled ? 1.f : 0.f, 0.f})
            o.push_back(x);
    }
    if (env.scenario != Env::S_TOWER) {
        uint32_t reached = 0, alive[3] = {0, 0, 0};
        env.agentReachedExit.resize(size_t(env.numAgents), false);
        for (int i = 0; i < env.numAgents; ++i) reached |= env.agentReachedExit[size_t(i)] ? (1u << i) : 0u;
        if (env.scenario == Env::S_REARRANGE) reached = uint32_t(env.maxMatchingObjects);
        if (env.scenario == Env::S_HEX_EXPLORE) alive[0] = env.exploreRewardAlive ? 1u : 0u;
        if (env.scenario == Env::S_HEX_MEMORY) {
            reached = uint32_t(env.goodObjectsCollected);
            for (size_t r = 0; r < env.memoryObjects.size() && r < 96; ++r)
                if (env.memoryObjects[r].alive) alive[r >> 5] |= 1u << (r & 31);
        }
        for (size_t r = 0; r < env.rewardSpawnPositions.size() && r < 96; ++r) {
            const Voxel *v = env.vg.grid.get(env.rewardSpawnPositions[r]);
            if (v && v->rewardObject == int(r)) alive[r >> 5] |= 1u << (r & 31);
        }
        o.push_back(float(env.solved)); o.push_back(float(reached));
        for (int w = 0; w < 3; ++w) o.push_back(float(alive[w] & 0xffffffu)), o.push_back(float(alive[w] >> 24));
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::memcpy(out, o.data(), o.size() * sizeof(float));
    return int(o.size());
}

// Rearrange: [0] = items n, then per item 5 ints (shape, palette colour, offset3); then objects m and per object 2 ints
// (shape, palette colour); then the work centre (3 ints) -- lets a test script a solving policy
int orc_get_arrangement(void *p, int envIdx, int32_t *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(envIdx)];
    std::vector<int32_t> o;
    o.push_back(int(env.arrangement.size()));
    for (auto &it : env.arrangement)
        for (int x : {it.shape, paletteIndex(it.color), int(it.offset.x), int(it.offset.y), int(it.offset.z)}) o.push_back(x);
    o.push_back(int(env.arrangementObjects.size()));
    for (int obj : env.arrangementObjects) { o.push_back(env.objects[size_t(obj)].mesh); o.push_back(env.objects[size_t(obj)].color); }
    for (int x : {int(env.rightCenter.x), int(env.rightCenter.y), int(env.rightCenter.z)}) o.push_back(x);
    if (int(o.size()) > cap) return -int(o.size());
    std::memcpy(out, o.data(), o.size() * sizeof(int32_t));
    return int(o.size());
}

// the restated layout helpers, same sequence and layout as ref_layout_utils_case (oracle/ref_shim/ref_shim.cpp)
int orc_layout_utils_case(unsigned seed, int32_t *out, int cap) {
    Env env("ObstaclesEasy", 1, {});
    Rng rng(seed);
    auto fr = [&](float lo, float hi) { return lo + (hi - lo) * frand(rng); };
    Boxes boxes;
    for (int i = 0; i < 5; ++i) {
        const int x = randRange(-5, 20, rng), y = randRange(0, 4, rng), z = randRange(-5, 20, rng);
        const int x1 = x + randRange(0, 9, rng), y1 = y + randRange(0, 3, rng), z1 = z + randRange(0, 9, rng);
        boxes.push_back(BoundingBox{VoxelCoords(x, y, z), VoxelCoords(x1, y1, z1)});
    }
    env.addBoundingBoxes(boxes, VOXEL_SOLID | VOXEL_OPAQUE, GREY, 1.0f);
    env.addBoundingBoxes(boxes, VOXEL_SOLID, DARK_GREY, 2.0f);
    env.addBoundingBoxes(boxes, VOXEL_OPAQUE, ORANGE, 1.0f);
    for (int i = 0; i < 4; ++i) {
        const int x = randRange(0, 20, rng), z = randRange(0, 20, rng);
        const int y = randRange(1, 3, rng), x1 = x + randRange(0, 6, rng), z1 = z + randRange(1, 6, rng);
        env.addTerrain(i % 2 ? TERRAIN_LAVA : TERRAIN_EXIT, BoundingBox{VoxelCoords(x, y, z), VoxelCoords(x1, 2, z1)});
    }
    for (int i = 0; i < 4; ++i) {
        const float sx = fr(0.1f, 9), sy = fr(0.0001f, 2), sz = fr(0.1f, 9);
        const float tx = fr(-20, 20), ty = fr(-1, 3), tz = fr(-20, 20);
        env.addStaticCollidingBox({sx, sy, sz}, {tx, ty, tz}, BLUE);
    }
    for (int i = 0; i < 3; ++i) {
        { const float x = fr(-20, 20), y = fr(0, 3), z = fr(-20, 20); const float k = fr(0.5f, 2.5f); env.addMemoryShape(Env::SHAPE_DIAMOND, GREEN, {x, y, z}, Vec3{0.17f, 0.45f, 0.17f} * k, false, true); }
        { const float x = fr(-20, 20), y = fr(0, 3), z = fr(-20, 20); const float k = fr(0.5f, 1.5f); env.addMemoryShape(Env::SHAPE_PILLAR, VIOLET, {x, y, z}, Vec3{0.5f, 2, 0.5f} * k, false, true); }
        { const float x = fr(-20, 20), y = fr(0, 3), z = fr(-20, 20); const float k = fr(0.5f, 1.5f); env.addMemoryShape(Env::SHAPE_SPHERE, RED, {x, y, z}, Vec3{0.75f, 0.75f, 0.75f} * k, false, true); }
    }
    std::vector<int32_t> o;
    auto bits = [](float f) { int32_t u; std::memcpy(&u, &f, 4); return u; };
    for (int t = 0; t < 5; ++t) o.push_back(int(env.drawables[t].size()));
    for (int t = 0; t < 5; ++t)
        for (auto &d : env.drawables[t]) {
            for (int i = 0; i < 16; ++i) o.push_back(bits((&d.model.c[0][0])[i]));
            const unsigned c = unsigned(allColors[d.color]);
            for (float f : {float((c >> 16) & 255) / 255.0f, float((c >> 8) & 255) / 255.0f, float(c & 255) / 255.0f}) o.push_back(bits(f));
        }
    o.push_back(int(env.colliders.size()));
    for (auto &c : env.colliders)
        for (float f : {c.c.x, c.c.y, c.c.z, c.h.x, c.h.y, c.h.z}) o.push_back(bits(f));
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}
// the restated pick-up / put-down logic (Env::onInteractAction), same scripted scene and layout as ref_stacking_case
int orc_stacking_case(const int *solid, int nSolid, const int *objVoxels, int nObj, int nAgents, const float *script, int nEvents, int32_t *out, int cap) {
    Env env("ObstaclesEasy", nAgents, {});  // a scenario whose stacking callbacks are the defaults (canPlaceObject: true)
    env.vg.reset();
    env.agents.assign(size_t(nAgents), Agent{});
    for (auto &a : env.agents) a.pickupLocal = mul(mat4Translation({0.0f, -0.44f, -1.0f}), mat4Identity());
    env.carryingObject.assign(size_t(nAgents), -1);
    for (int i = 0; i < nSolid; ++i) env.vg.grid.set(VoxelCoords(solid[i * 3], solid[i * 3 + 1], solid[i * 3 + 2]), VoxelGridComponent::makeVoxel(VOXEL_SOLID | VOXEL_OPAQUE));
    std::vector<VoxelCoords> positions;
    for (int i = 0; i < nObj; ++i) positions.emplace_back(objVoxels[i * 3], objVoxels[i * 3 + 1], objVoxels[i * 3 + 2]);
    env.addObjects(positions);
    std::vector<int32_t> o;
    auto bits = [](float f) { int32_t u; std::memcpy(&u, &f, 4); return u; };
    for (int ev = 0; ev < nEvents; ++ev) {
        const float *e = script + size_t(ev) * 33;
        const int ai = int(e[0]);
        std::memcpy(&env.agents[size_t(ai)].objectT.c[0][0], e + 1, 64);
        std::memcpy(&env.agents[size_t(ai)].cameraLocal.c[0][0], e + 17, 64);
        env.onInteractAction(ai);
        for (int k = 0; k < nObj; ++k) {
            const MovableObject &ob = env.objects[size_t(k)];
            const Vec3 t = translationOf(env.objectAbs(k)), sc = scalingOf(ob.local);
            for (float f : {t.x, t.y, t.z, sc.x, sc.y, sc.z}) o.push_back(bits(f));
            o.push_back(ob.parentAgent); o.push_back(env.colliders[size_t(ob.collider)].enabled ? 1 : 0);
        }
        for (int a = 0; a < nAgents; ++a) o.push_back(env.carryingObject[size_t(a)]);
        std::vector<std::array<int32_t, 4>> occ;
        for (auto &kv : env.vg.grid.getHashMap())
            if (kv.second.physicsObject >= 0) occ.push_back({kv.first.x, kv.first.y, kv.first.z, kv.second.physicsObject});
        std::sort(occ.begin(), occ.end());
        o.push_back(int(occ.size()));
        for (auto &r : occ) for (int v : r) o.push_back(v);
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}
// the restated layout pipeline, same case and layout as ref_voxel_layout_case (oracle/ref_shim/ref_shim.cpp)
int orc_voxel_layout_case(int type, unsigned seed, int rotate, int drawWalls, const float *params9, int32_t *out, int cap) {
    FloatParams fp{{"obstaclesMinGap", params9[0]}, {"obstaclesMaxGap", params9[1]}, {"obstaclesMinLava", params9[2]}, {"obstaclesMaxLava", params9[3]},
                   {"obstaclesMinHeight", params9[4]}, {"obstaclesMaxHeight", params9[5]}, {"verticalLookLimitRad", params9[6]}, {"episodeLengthSec", params9[7]},
                   {"obstaclesNumAllowedMaxDifficulty", params9[8]}};
    Rng rng(seed);
    auto levelRoot = std::make_unique<Node>();
    StartPlatform start(levelRoot.get(), rng, fp);
    start.init(); start.generate();
    std::unique_ptr<Platform> p;
    const int walls = 4 | 8, w = rotate ? -1 : start.width;
    switch (type) {
        case 1: p = std::make_unique<WallPlatform>(start.nextPlatformAnchor, rng, walls, fp, w); break;
        case 2: p = std::make_unique<LavaPlatform>(start.nextPlatformAnchor, rng, walls, fp, w); break;
        case 3: p = std::make_unique<StepPlatform>(start.nextPlatformAnchor, rng, walls, fp, w); break;
        case 4: p = std::make_unique<GapPlatform>(start.nextPlatformAnchor, rng, walls, fp, w); break;
        default: p = std::make_unique<ExitPlatform>(start.nextPlatformAnchor, rng, fp, w); break;
    }
    p->init();
    if (rotate == 1) p->rotateCCW(start.width); else if (rotate == 2) p->rotateCW(start.width);
    p->generate();
    VoxelGridComponent vg(100, 0, 0, 0, 1);
    vg.addPlatform(start, LAYOUT_DEFAULT, DARK_GREY, bool(drawWalls));
    vg.addPlatform(*p, VERY_LIGHT_BLUE, GREY, bool(drawWalls));
    const auto byType = vg.toBoundingBoxes();
#define BX(v) (v).x
#define BY(v) (v).y
#define BZ(v) (v).z

    std::vector<int32_t> o;
    o.push_back(int(byType.size()));
    for (auto &kv : byType) {
        o.push_back(int(kv.first.type)); o.push_back(int(kv.first.color)); o.push_back(int(kv.second.size()));
        for (auto &b : kv.second) for (int v : {BX(b.min), BY(b.min), BZ(b.min), BX(b.max), BY(b.max), BZ(b.max)}) o.push_back(v);
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());

#undef BX
#undef BY
#undef BZ
}
// the restated platforms (orc_level.hpp), same case and layout as ref_platform_case (oracle/ref_shim/ref_shim.cpp)
int orc_platform_case(int type, unsigned seed, int walls, int w, int l, int rotate, int prevWidth, const float *params9, int nObjects, int nAgents, int32_t *out, int cap) {
    FloatParams fp{{"obstaclesMinGap", params9[0]}, {"obstaclesMaxGap", params9[1]}, {"obstaclesMinLava", params9[2]}, {"obstaclesMaxLava", params9[3]},
                   {"obstaclesMinHeight", params9[4]}, {"obstaclesMaxHeight", params9[5]}, {"verticalLookLimitRad", params9[6]}, {"episodeLengthSec", params9[7]},
                   {"obstaclesNumAllowedMaxDifficulty", params9[8]}};
    Rng rng(seed);
    auto sceneRoot = std::make_unique<Node>();
    auto anchorOwner = std::make_unique<Node>();
    Node *anchor = anchorOwner.get();
    anchor->parent = sceneRoot.get();
    anchor->local = mul(mat4Translation({3, 1, 2}), anchor->local);
    std::unique_ptr<Platform> p;
    switch (type) {
        case 0: p = std::make_unique<EmptyPlatform>(anchor, rng, walls, fp, w); break;
        case 1: p = std::make_unique<WallPlatform>(anchor, rng, walls, fp, w); break;
        case 2: p = std::make_unique<LavaPlatform>(anchor, rng, walls, fp, w); break;
        case 3: p = std::make_unique<StepPlatform>(anchor, rng, walls, fp, w); break;
        case 4: p = std::make_unique<GapPlatform>(anchor, rng, walls, fp, w); break;
        case 5: p = std::make_unique<StartPlatform>(anchor, rng, fp, w); break;
        case 6: p = std::make_unique<ExitPlatform>(anchor, rng, fp, w); break;
        default: p = std::make_unique<TransitionPlatform>(anchor, rng, walls, fp, l, w); break;
    }
    p->init();
    if (rotate == 1) p->rotateCCW(prevWidth); else if (rotate == 2) p->rotateCW(prevWidth);
    p->generate();
#define BX(v) (v).x
#define BY(v) (v).y
#define BZ(v) (v).z

    std::vector<int32_t> o;
    auto pushBox = [&](const BoundingBox &b) { for (int v : {BX(b.min), BY(b.min), BZ(b.min), BX(b.max), BY(b.max), BZ(b.max)}) o.push_back(v); };
    for (int v : {p->length, p->height, p->width, int(p->isMaxDifficulty()), p->requiresMovableBoxesToTraverse()}) o.push_back(v);
    o.push_back(int(p->layoutBoxes.size()));
    for (auto &b : p->layoutBoxes) pushBox(b.boundingBox());
    o.push_back(int(p->wallBoxes.size()));
    for (auto &b : p->wallBoxes) pushBox(b.boundingBox());
    o.push_back(int(p->terrainBoxes.size()));
    for (auto &kv : p->terrainBoxes) { o.push_back(int(kv.first)); o.push_back(int(kv.second.size())); for (auto &b : kv.second) pushBox(b.boundingBox()); }
    pushBox(p->platformBoundingBox());

    const auto objs = p->generateObjectPositions(nObjects);
    o.push_back(int(objs.size()));
    for (auto &c : objs) for (int v : {int(c.x), int(c.y), int(c.z)}) o.push_back(v);
    const auto spawns = p->agentSpawnPoints(nAgents);
    o.push_back(int(spawns.size()));
    for (auto &c : spawns) for (float f : {c.x, c.y, c.z}) { int32_t u; std::memcpy(&u, &f, 4); o.push_back(u); }
    if (p->nextPlatformAnchor) {
        const Vec3 t = translationOf(p->nextPlatformAnchor->absolute());
        for (float f : {t.x, t.y, t.z}) { int32_t u; std::memcpy(&u, &f, 4); o.push_back(u); }
    }
#undef BX
#undef BY
#undef BZ
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}
// the scene-graph conventions the restatement uses (see ref_scenegraph_case in oracle/ref_shim/ref_shim.cpp for the scenario code it mirrors)
void orc_scenegraph_case(const float *ps, float angle, const float *pt, const float *cs, const float *ct, const float *fs, const float *ft,
                         const float *rs, const float *rt, float *out48) {
    const Mat4 parentLocal = mul(mat4Translation({pt[0], pt[1], pt[2]}), mul(mat4RotationY(angle), mul(mat4Scaling({ps[0], ps[1], ps[2]}), mat4Identity())));
    const Mat4 childLocal = mul(mat4Translation({ct[0], ct[1], ct[2]}), mul(mat4Identity(), mat4Scaling({cs[0], cs[1], cs[2]})));
    const Mat4 childAbs = mul(parentLocal, childLocal);
    std::memcpy(out48, &childAbs.c[0][0], 64);
    std::memcpy(out48 + 16, &childAbs.c[0][0], 64);
    const Mat4 root = mul(mat4Translation({rt[0], rt[1], rt[2]}), mul(mat4Scaling({rs[0], rs[1], rs[2]}), mat4Identity()));
    const Mat4 freeAbs = mul(mat4Translation({ft[0], ft[1], ft[2]}), mul(mat4Scaling({fs[0], fs[1], fs[2]}), mat4Identity()));
    const Mat4 local = mul(inverted(root), freeAbs);  // setParentKeepTransformation
    const Mat4 abs = mul(root, local);
    std::memcpy(out48 + 32, &abs.c[0][0], 64);
}
// One mv_debug_kcc case list (same layouts, include/megaverse_b200.h) through the oracle's own queries over the FULL collider list: no
// envelope, no candidate cap, so out_i8[0] is the number of enabled colliders other than the agent and out_i8[1] is 0.  Arguments are
// trusted (the tests build them).
constexpr int kKccMaxObjects = 128, kKccMaxAgents = 8;  // the layouts' row counts: the engine's MV_MAX_OBJECTS and MV_MAX_AGENTS
void orc_kcc_case(const int32_t *hdr8, const float *boxes10, const float *agents3, const float *query20, int n, int32_t *out_i8, float *out_f16) {
    for (int cs = 0; cs < n; ++cs) {
        const int32_t *hd = hdr8 + size_t(cs) * 8;
        const int nsPre = hd[0], ns = hd[1], no = hd[2], A = hd[3], mode = hd[4], agent = hd[5];
        const float *q = query20 + size_t(cs) * 20;
        std::vector<Collider> cols;
        auto box = [&](int row, bool isStatic) {
            const float *b = boxes10 + (size_t(cs) * 2 * kKccMaxObjects + size_t(row)) * 10;
            Collider c;
            c.c = {b[0], b[1], b[2]}; c.h = {b[3], b[4], b[5]}; c.enabled = b[6] != 0.0f;
            if (isStatic && b[7] != 0.0f) { c.rotated = true; c.ax = b[8]; c.az = b[9]; }
            cols.push_back(c);
        };
        for (int j = 0; j < nsPre; ++j) box(j, true);
        for (int j = 0; j < no; ++j) box(kKccMaxObjects + j, false);
        for (int j = nsPre; j < ns; ++j) box(j, true);
        for (int a = 0; a < A; ++a) {
            const float *p = agents3 + (size_t(cs) * kKccMaxAgents + size_t(a)) * 3;
            Collider c;
            c.kind = 1; c.c = (mode == 2 && a == agent) ? Vec3{q[0], q[1], q[2]} : Vec3{p[0], p[1], p[2]};
            cols.push_back(c);
        }
        const int self = ns + no + agent;
        int32_t *oi = out_i8 + size_t(cs) * 8;
        float *of = out_f16 + size_t(cs) * 16;
        for (int j = 0; j < 8; ++j) oi[j] = 0;
        for (int j = 0; j < 16; ++j) of[j] = 0.0f;
        for (int j = 0; j < int(cols.size()); ++j) oi[0] += j != self && cols[size_t(j)].enabled;
        oi[3] = oi[4] = -1;
        if (mode == 0) {
            const SweepHit r = convexSweep(cols, self, {q[0], q[1], q[2]}, {q[3], q[4], q[5]}, {q[6], q[7], q[8]}, q[9]);
            oi[2] = r.hit;
            if (r.hit) { oi[3] = r.index; oi[4] = r.feature; }
            of[0] = r.fraction; of[1] = r.normal.x; of[2] = r.normal.y; of[3] = r.normal.z;
        } else if (mode == 1) {
            KCC k;
            k.pos = {q[0], q[1], q[2]};
            int idx = -1;
            oi[2] = k.recoverFromPenetration(cols, self, &idx);
            if (oi[2]) {  // the push-out itself, as recoverFromPenetration forms it before adding it to the position
                Vec3 nrm;
                const float dist = capsuleDistance(cols[size_t(idx)], {q[0], q[1], q[2]}, nrm);
                const Vec3 delta = nrm * (-dist);
                oi[3] = idx; of[0] = delta.x; of[1] = delta.y; of[2] = delta.z;
            }
        } else {
            KCC k;
            k.pos = {q[0], q[1], q[2]}; k.horizontalVelocity = {q[3], q[4], q[5]};
            k.verticalVelocity = q[6]; k.verticalOffset = q[7]; k.currentStepOffset = q[8]; k.jumpSpeed = q[9];
            k.jumpAxis = {q[10], q[11], q[12]};
            k.wasOnGround = q[13] != 0.0f; k.wasJumping = q[14] != 0.0f;
            k.maxSlopeCosine = q[16];
            k.playerStep(cols, self, q[15]);
            oi[2] = k.wasOnGround; oi[5] = k.wasJumping;
            of[0] = k.pos.x; of[1] = k.pos.y; of[2] = k.pos.z;
            of[3] = k.horizontalVelocity.x; of[4] = k.horizontalVelocity.y; of[5] = k.horizontalVelocity.z;
            of[6] = k.verticalVelocity; of[7] = k.verticalOffset; of[8] = k.currentStepOffset; of[9] = k.jumpSpeed;
        }
    }
}

// colour tables of the restatement, same layout as ref_color_tables (oracle/ref_shim/ref_shim.cpp)
int orc_color_tables(unsigned *out, int cap) {
    std::vector<unsigned> o{unsigned(numColors), unsigned(numAgentColors), unsigned(numObjectColors), unsigned(numLayoutColors)};
    for (int i = 0; i < numColors; ++i) o.push_back(unsigned(allColors[i]));
    for (int i = 0; i < numAgentColors; ++i) o.push_back(unsigned(agentColors[i]));
    for (int i = 0; i < numObjectColors; ++i) o.push_back(unsigned(objectColors[i]));
    for (int i = 0; i < numLayoutColors; ++i) o.push_back(unsigned(layoutColors[i]));
    for (int i = 0; i < numColors; ++i) {
        const unsigned c = unsigned(allColors[i]);
        for (float f : {float((c >> 16) & 255) / 255.0f, float((c >> 8) & 255) / 255.0f, float(c & 255) / 255.0f}) { unsigned u; std::memcpy(&u, &f, 4); o.push_back(u); }
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}
// the Perlin restatement (orc_level.hpp), same call as ref_perlin
void orc_perlin(unsigned seed, int n, const double *xy, int octaves, double *out) {
    const PerlinNoise perlin(seed);
    for (int i = 0; i < n; ++i) out[i] = perlin.accumulatedOctaveNoise2D_0_1(xy[2 * i], xy[2 * i + 1], octaves);
}
// the honeycomb maze restatement, same layout as ref_honeycomb_maze (oracle/ref_shim/ref_shim.cpp)
int orc_honeycomb_maze(int size, unsigned seed, double *out, int cap) {
    HoneyCombMaze maze(size);
    std::mt19937 gen(seed);
    maze.initialiseGraph();
    maze.generate(gen);
    std::vector<double> o;
    o.push_back(double(maze.adjacency.size()));
    for (size_t c = 0; c < maze.adjacency.size(); ++c) {
        o.push_back(maze.cellCenters[c].first); o.push_back(maze.cellCenters[c].second); o.push_back(double(maze.adjacency[c].size()));
        for (auto &e : maze.adjacency[c])
            for (double v : {double(e.cell), e.border[0], e.border[1], e.border[2], e.border[3]}) o.push_back(v);
    }
    for (double v : maze.coordinateBounds()) o.push_back(v);
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}

// solid/object occupancy: sorted list of (x,y,z,flags) with flags bit0 solid, bit1 opaque, bit2 holds object; terrain in bits 8..
int orc_get_voxels(void *p, int envIdx, int32_t *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(envIdx)];
    std::vector<std::array<int32_t, 4>> v;
    for (auto &kv : env.vg.grid.getHashMap()) {
        const int flags = int(kv.second.voxelType) | (kv.second.physicsObject >= 0 ? 4 : 0) | (int(kv.second.terrain) << 8);
        if (flags == 0) continue;  // an entry that became empty again is indistinguishable from no entry
        v.push_back({kv.first.x, kv.first.y, kv.first.z, flags});
    }
    std::sort(v.begin(), v.end());
    if (int(v.size()) * 4 > cap) return -int(v.size()) * 4;
    for (size_t i = 0; i < v.size(); ++i) std::memcpy(out + i * 4, v[i].data(), 16);
    return int(v.size()) * 4;
}

// instances of one env in draw order: per instance 18 floats (mesh, color, 16 model matrix column-major); view matrices
int orc_get_instances(void *p, int envIdx, float *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(envIdx)];
    const auto inst = env.instances();
    if (int(inst.size()) * 18 > cap) return -int(inst.size()) * 18;
    for (size_t i = 0; i < inst.size(); ++i) {
        out[i * 18] = float(inst[i].mesh); out[i * 18 + 1] = float(inst[i].color);
        std::memcpy(out + i * 18 + 2, &inst[i].model.c[0][0], 64);
    }
    return int(inst.size()) * 18;
}
void orc_get_view(void *p, int envIdx, int agent, float *out16) {
    const Mat4 m = static_cast<OrcVec *>(p)->envs[size_t(envIdx)]->viewMatrix(agent);
    std::memcpy(out16, &m.c[0][0], 64);
}
// stand-alone rasteriser entry: render given instances + view (for renderer-only parity tests)
void orc_render_instances(const float *view16, const float *inst18, int n, int w, int h, uint8_t *rgba, float *depth) {
    Mat4 view;
    std::memcpy(&view.c[0][0], view16, 64);
    std::vector<Instance> inst(static_cast<size_t>(n));
    for (int i = 0; i < n; ++i) {
        inst[size_t(i)].mesh = int(inst18[i * 18]); inst[size_t(i)].color = int(inst18[i * 18 + 1]);
        std::memcpy(&inst[size_t(i)].model.c[0][0], inst18 + i * 18 + 2, 64);
    }
    renderView(view, inst, w, h, rgba, depth);
}
// mesh tables (float bit patterns) so tests can compare the product's own tables with the reference's Magnum
int orc_get_mesh(int type, uint32_t *vtx, int capV, uint16_t *idx, int capI) {
    const MeshRef m = meshRef(type);
    if (m.nv * 6 > capV || m.ni > capI) return -1;
    std::memcpy(vtx, m.vtx, size_t(m.nv) * 24);
    std::memcpy(idx, m.idx, size_t(m.ni) * 2);
    return m.nv * 65536 + m.ni;
}
// iteration order of a REAL std::unordered_set<VoxelCoords> (the reference's objectsInBuildingZone type) after a sequence
// of ops {op(0 insert, 1 erase, 2 clear), x, y, z}: pins the product's libstdc++-order emulation (csrc/bzset.h)
int orc_unordered_set_order(const int32_t *ops, int nops, int32_t *out, int cap) {
    std::unordered_set<VoxelCoords, VoxelHash> s;
    for (int i = 0; i < nops; ++i) {
        const int32_t *o = ops + i * 4;
        if (o[0] == 0) s.insert({o[1], o[2], o[3]});
        else if (o[0] == 1) s.erase({o[1], o[2], o[3]});
        else s.clear();
    }
    int n = 0;
    for (auto &v : s) {
        if (n * 3 + 3 > cap) return -1;
        out[n * 3] = v.x; out[n * 3 + 1] = v.y; out[n * 3 + 2] = v.z;
        ++n;
    }
    return n;
}
// restated math, exposed so tests/test_ref_shim.py can pin it against the real Magnum / util headers (oracle/_ref)
static Mat4 loadM(const float *p) { Mat4 m; std::memcpy(&m.c[0][0], p, 64); return m; }
void orc_mat4_mul(const float *a, const float *b, float *out) { const Mat4 m = mul(loadM(a), loadM(b)); std::memcpy(out, &m.c[0][0], 64); }
void orc_mat4_inverted(const float *a, float *out) { const Mat4 m = inverted(loadM(a)); std::memcpy(out, &m.c[0][0], 64); }
void orc_mat4_rotation(float angle, const float *ax, float *out) { const Mat4 m = mat4Rotation(angle, {ax[0], ax[1], ax[2]}); std::memcpy(out, &m.c[0][0], 64); }
void orc_mat4_rotation_x(float angle, float *out) { const Mat4 m = mat4RotationX(angle); std::memcpy(out, &m.c[0][0], 64); }
void orc_mat4_rotation_y(float angle, float *out) { const Mat4 m = mat4RotationY(angle); std::memcpy(out, &m.c[0][0], 64); }
void orc_mat4_scaling_of(const float *a, float *out3) { const Vec3 s = scalingOf(loadM(a)); out3[0] = s.x; out3[1] = s.y; out3[2] = s.z; }
void orc_mat4_transform_point(const float *a, const float *p, float *out3) { const Vec3 r = transformPoint(loadM(a), {p[0], p[1], p[2]}); out3[0] = r.x; out3[1] = r.y; out3[2] = r.z; }
void orc_vec3_normalized(const float *v, float *out3) { const Vec3 r = mgNormalized({v[0], v[1], v[2]}); out3[0] = r.x; out3[1] = r.y; out3[2] = r.z; }
unsigned long long orc_voxel_hash(int x, int y, int z) { return VoxelHash{}(VoxelCoords{x, y, z}); }
void orc_rng_stream(unsigned seed, int lo, int hi, int n, int *ints, float *floats) {
    Rng rng(seed);
    for (int i = 0; i < n; ++i) ints[i] = randRange(lo, hi, rng);
    for (int i = 0; i < n; ++i) floats[i] = frand(rng);
}
int orc_voxel_grid_order(const int *xyz, int n, int *out_xyz) {
    VoxelGrid grid(100, {0, 0, 0}, 1);
    for (int i = 0; i < n; ++i) grid.set({xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2]}, Voxel{});
    int k = 0;
    const auto copy = grid.getHashMap();
    for (auto &kv : copy) { out_xyz[k * 3] = kv.first.x; out_xyz[k * 3 + 1] = kv.first.y; out_xyz[k * 3 + 2] = kv.first.z; ++k; }
    return k;
}
void orc_to_voxel(float x, float y, float z, int32_t *out) { const VoxelCoords v = toVoxel({x, y, z}); out[0] = v.x; out[1] = v.y; out[2] = v.z; }
// libstdc++ stream probe (SURVEY.md Appendix C): mt19937(42) first raw, uniform_int{0,9}, then frand
void orc_rng_probe(double *out3) {
    Rng raw(42);
    out3[0] = double(raw());
    Rng r(42);
    out3[1] = double(std::uniform_int_distribution<>{0, 9}(r));
    out3[2] = double(frand(r));
}
int orc_max_threads() { return int(std::thread::hardware_concurrency()); }


// ---- scenario pin (tests/test_ref_shim.py): one env driven tick by tick beside the reference's real scenario sources
// (oracle/ref_shim/scen_shim.cpp).  Layouts match ref_scen_*.
static uint32_t fbits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
void orc_scen_reset(void *p, int e) { static_cast<OrcVec *>(p)->envs[size_t(e)]->reset(); }
void orc_scen_step(void *p, int e, const int *actions) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    for (int i = 0; i < env.numAgents; ++i) env.setAction(i, actions[i]);
    env.step();
}
// test hook: put an agent somewhere else (btKinematicCharacterController::warp, as FallDetectionComponent does) so that scripted
// trajectories reach the objects, boxes and rewards quickly; the reference-side puppets follow through orc_scen_poses
void orc_scen_warp(void *p, int e, int agent, float x, float y, float z, float yaw) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    env.agents[size_t(agent)].kcc.warp({x, y, z});
    env.agents[size_t(agent)].kcc.basis = mat3FromQuat(quatAxisAngle({0, 1, 0}, yaw));  // as DefaultKinematicAgent's constructor turns it
    env.colliders[size_t(env.agentColliderBase + agent)].c = env.agents[size_t(agent)].kcc.pos;
}
int orc_scen_undefined_spawn(void *p, int e) { return static_cast<OrcVec *>(p)->envs[size_t(e)]->undefinedSpawn ? 1 : 0; }
void orc_scen_spawns(void *p, int e, uint32_t *out) {  // per agent: DefaultKinematicAgent's startingPosition xyz, rotationRad
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    for (int i = 0; i < env.numAgents; ++i) {
        const Agent &a = env.agents[size_t(i)];
        out[4 * i] = fbits(a.spawnPos.x), out[4 * i + 1] = fbits(a.spawnPos.y), out[4 * i + 2] = fbits(a.spawnPos.z), out[4 * i + 3] = fbits(a.spawnRot);
    }
}
void orc_scen_poses(void *p, int e, float *out) {  // per agent: objectT[16] cameraLocal[16] onGround (column-major, as Magnum stores)
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    for (int i = 0; i < env.numAgents; ++i) {
        const Agent &a = env.agents[size_t(i)];
        std::memcpy(out + i * 33, &a.objectT, 64);
        std::memcpy(out + i * 33 + 16, &a.cameraLocal, 64);
        out[i * 33 + 32] = a.kcc.onGround() ? 1.0f : 0.0f;
    }
}
void orc_scen_teleports(void *p, int e, uint32_t *out) {  // per agent: (count, last target xyz)
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    for (int i = 0; i < env.numAgents; ++i) out[4 * i] = 0, out[4 * i + 1] = out[4 * i + 2] = out[4 * i + 3] = fbits(0.0f);
    for (auto &[i, t] : env.teleportLog) { ++out[4 * i]; out[4 * i + 1] = fbits(t.x), out[4 * i + 2] = fbits(t.y), out[4 * i + 3] = fbits(t.z); }
}
int orc_scenario_dump(void *p, int e, uint32_t *out, int cap) {
    Env &env = *static_cast<OrcVec *>(p)->envs[size_t(e)];
    std::vector<uint32_t> o;
    o.push_back(fbits(env.episodeLengthSec()));
    o.push_back(env.done ? 1u : 0u);
    o.push_back(fbits(env.currEpisodeSec));
    o.push_back(uint32_t(env.numAgents));
    for (int i = 0; i < env.numAgents; ++i) {
        o.push_back(fbits(env.lastReward[size_t(i)]));
        o.push_back(fbits(env.totalReward[size_t(i)]));
        o.push_back(fbits(env.trueObjective(i)));
    }
    const auto inst = env.instances();
    o.push_back(uint32_t(inst.size()));
    for (auto &in : inst) {
        o.push_back(uint32_t(in.mesh));
        o.push_back(uint32_t(allColors[in.color]));
        const float *m = reinterpret_cast<const float *>(&in.model);
        for (int k = 0; k < 16; ++k) o.push_back(fbits(m[k]));
    }
    o.push_back(uint32_t(env.agentColliderBase));
    for (int c = 0; c < env.agentColliderBase; ++c) {
        const Collider &col = env.colliders[size_t(c)];
        o.push_back(fbits(col.c.x)), o.push_back(fbits(col.c.y)), o.push_back(fbits(col.c.z));
        o.push_back(fbits(col.h.x)), o.push_back(fbits(col.h.y)), o.push_back(fbits(col.h.z));
        o.push_back(fbits(col.rotated ? col.ax : 1.0f)), o.push_back(fbits(col.rotated ? col.az : 0.0f));
        o.push_back(col.enabled ? 1u : 0u);
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}

// ---- fragment / vertex stage pieces for the shader pin (tests/test_ref_shim.py, oracle/ref_shim/shade_shim.cpp)
void orc_shade(int n, const float *P3, const float *N3, const float *diffuse3, float *out3, uint8_t *outUnorm3) {
    for (int i = 0; i < n; ++i) {
        float Lo[3];
        shadeFragment(P3 + 3 * i, N3 + 3 * i, diffuse3 + 3 * i, Lo);
        for (int c = 0; c < 3; ++c) { out3[3 * i + c] = Lo[c]; outUnorm3[3 * i + c] = toUnorm8(Lo[c]); }
    }
}
void orc_normal_matrix(const float *mv16, float *out9) {  // column-major 3x3, as uber.vert's normal_mat
    Mat4 mv;
    std::memcpy(&mv.c[0][0], mv16, 64);
    float nm[3][3];
    normalMatrix(mv, nm);
    std::memcpy(out9, nm, 36);
}

// ---- the analytic narrow phase on its own (tests/test_cpu.py: the sweep against its definition through the distance function)
// collider8: kind, cx, cy, cz, hx, hy, hz, yaw (kind 0 = box turned by yaw about Y, 1 = another agent's capsule)
static Collider colliderFrom(const float *c8) {
    Collider c;
    c.kind = int(c8[0]);
    c.c = {c8[1], c8[2], c8[3]};
    c.h = {c8[4], c8[5], c8[6]};
    if (c.kind == 0 && c8[7] != 0.0f) { c.rotated = true; c.ax = crcos(c8[7]); c.az = -crsin(c8[7]); }
    return c;
}
int orc_sweep_case(const float *collider8, const float *from3, const float *to3, float *t, float *n3) {
    const Collider c = colliderFrom(collider8);
    const Vec3 f{from3[0], from3[1], from3[2]}, to{to3[0], to3[1], to3[2]};
    Vec3 n{0, 0, 0};
    float tt = 1.0f;
    const bool hit = !sweepBroadphaseMiss(c, f, to) && sweepNarrow(c, f, to - f, tt, n);
    *t = tt; n3[0] = n.x, n3[1] = n.y, n3[2] = n.z;
    return hit ? 1 : 0;
}
float orc_capsule_distance(const float *collider8, const float *p3, float *n3) {
    const Collider c = colliderFrom(collider8);
    Vec3 n{0, 0, 0};
    const float d = capsuleDistance(c, {p3[0], p3[1], p3[2]}, n);
    n3[0] = n.x, n3[1] = n.y, n3[2] = n.z;
    return d;
}
}  // extern "C"
