// Host-side procedural level generation (product code).  See levelgen.hpp.
//
// Reference behaviour reproduced here (file:line under /root/reference):
//   Env::reset reseed                         src/libs/env/src/env.cpp:61-62
//   TowerBuildingScenario::reset / platform   src/libs/scenarios/src/scenario_tower_building.cpp:19-78,129-154
//   EmptyPlatform::generate (floor + walls)   src/libs/scenarios/include/scenarios/platforms.hpp:165-188,325-329
//   VoxelGridComponent::addPlatform           src/libs/scenarios/include/scenarios/component_voxel_grid.hpp:73-106
//   greedy voxel -> box merge                 src/libs/scenarios/include/scenarios/component_voxel_grid.hpp:108-187
//   addBoundingBoxes / addTerrain             src/libs/scenarios/src/layout_utils.cpp:17-68
//   DefaultScenario::spawnAgents              src/libs/scenarios/include/scenarios/scenario_default.hpp:80-97
//   colour tables                             src/libs/env/include/env/const.hpp:25-143
#include "levelgen.hpp"

#include <algorithm>
#include <array>
#include <cstdio>
#include <fstream>
#include <iterator>
#include <memory>
#include <cstring>
#include <set>
#include <stdexcept>
#include <unordered_map>
#include <unordered_set>

#include "hostmath.hpp"

namespace mv {

namespace {

// ---- colours -------------------------------------------------------------------------------------------------------
enum : uint32_t {
    C_YELLOW = 0xffdd3c, C_GREEN = 0x3bb372, C_LIGHT_GREEN = 0x50c878, C_BLUE = 0x2eb5d0, C_LIGHT_BLUE = 0xadd8e6, C_DARK_BLUE = 0x3a7fa6,
    C_DARK_NAVY = 0x2c3e50, C_ORANGE = 0xffb400, C_GREY = 0xb3b3b3, C_DARK_GREY = 0x555555, C_VERY_DARK_GREY = 0x222222, C_WHITE = 0xffffff,
    C_RED = 0xff0000, C_LIGHT_ORANGE = 0xffa770, C_VIOLET = 0xd468ee, C_LIGHT_PINK = 0xffe6e6, C_VL_YELLOW = 0xffffe6, C_VL_GREEN = 0xccffcc,
    C_VL_BLUE = 0xe6ecff, C_VL_GREY = 0xd9d9d9, C_VL_VIOLET = 0xf2e6ff, C_VL_ORANGE = 0xffebcc,
};
const uint32_t kPalette[22] = {C_YELLOW, C_GREEN, C_LIGHT_GREEN, C_BLUE, C_LIGHT_BLUE, C_DARK_BLUE, C_DARK_NAVY, C_ORANGE, C_GREY, C_DARK_GREY,
                               C_VERY_DARK_GREY, C_WHITE, C_RED, C_LIGHT_ORANGE, C_VIOLET, C_LIGHT_PINK, C_VL_YELLOW, C_VL_GREEN, C_VL_BLUE,
                               C_VL_GREY, C_VL_VIOLET, C_VL_ORANGE};
const uint32_t kLayoutColors[14] = {C_WHITE, C_VL_YELLOW, C_VL_GREEN, C_VL_BLUE, C_VL_GREY, C_VL_ORANGE, C_GREY, C_GREY, C_GREY, C_GREY,
                                    C_DARK_GREY, C_DARK_GREY, C_DARK_GREY, C_DARK_GREY};
int paletteIndex(uint32_t rgb) {
    for (int i = 0; i < 22; ++i)
        if (kPalette[i] == rgb) return i;
    return 0;
}

using Rng = std::mt19937;
int randRange(int low, int high, Rng &rng) { return std::uniform_int_distribution<>{low, high - 1}(rng); }
bool randomBool(Rng &rng) { return bool(randRange(0, 2, rng)); }
float frand(Rng &rng) { return std::uniform_real_distribution<float>{0, 1}(rng); }
uint32_t randomLayoutColor(Rng &rng) { return kLayoutColors[randRange(0, 14, rng)]; }
const uint32_t kObjectColors[14] = {C_YELLOW, C_GREEN, C_LIGHT_GREEN, C_BLUE, C_LIGHT_BLUE, C_DARK_BLUE, C_ORANGE, C_GREY, C_DARK_GREY, C_WHITE, C_RED,
                                    C_LIGHT_ORANGE, C_VIOLET, C_LIGHT_PINK};
uint32_t randomObjectColor(Rng &rng) { return kObjectColors[randRange(0, 14, rng)]; }  // const.hpp:96-119

// ---- sparse voxel map with the reference's hash (voxel_grid.hpp:39-49): iteration order must match -------------------
struct I3 { int x, y, z; };
inline uint32_t voxKey(int x, int y, int z) { return uint32_t(((x + 512) << 20) + ((y + 512) << 10) + (z + 512)); }
inline I3 voxUnkey(uint32_t k) { return {int(k >> 20) - 512, int((k >> 10) & 1023) - 512, int(k & 1023) - 512}; }
struct KeyHash { size_t operator()(uint32_t k) const noexcept { return size_t(k); } };
struct Vox { uint8_t type = 0, terrain = 0; uint32_t color = C_WHITE; };
using VoxMap = std::unordered_map<uint32_t, Vox, KeyHash>;

// ObjectStackingComponent::addDrawablesAndCollisions (component_object_stacking.hpp:170-198): a 0.39 box, MOVABLE_BOX colour,
// collision scale 1.15 / offset (0,-0.05,0) = collision class 0
void setStackingBox(MvObjInit &o, const I3 &v) {
    o.voxel[0] = int16_t(v.x); o.voxel[1] = int16_t(v.y); o.voxel[2] = int16_t(v.z);
    o.color = int16_t(paletteIndex(C_LIGHT_BLUE));
    o.scale[0] = o.scale[1] = o.scale[2] = 0.39f;
    o.meta = 0;
}

struct IBox { int mn[3], mx[3]; };  // max exclusive for platform boxes, inclusive for merged boxes (as in the reference)

void fillBox(VoxMap &g, const IBox &b, uint8_t type, uint32_t color) {
    for (int x = b.mn[0]; x < b.mx[0]; ++x)
        for (int y = b.mn[1]; y < b.mx[1]; ++y)
            for (int z = b.mn[2]; z < b.mx[2]; ++z) {
                Vox v; v.type = type; v.terrain = 0; v.color = color;
                g[voxKey(x, y, z)] = v;
            }
}
void fillTerrain(VoxMap &g, const IBox &b, int terrain) {
    for (int x = b.mn[0]; x < b.mx[0]; ++x)
        for (int y = b.mn[1]; y < b.mx[1]; ++y)
            for (int z = b.mn[2]; z < b.mx[2]; ++z) {
                const uint32_t k = voxKey(x, y, z);
                if (!g.count(k)) g[k] = Vox();
                g.find(k)->second.terrain |= uint8_t(terrain);
            }
}

struct MergedGroup { uint8_t type; uint32_t color; std::vector<IBox> boxes; };

// greedy expansion in -x,+x,-y,+y,-z,+z order, seeds visited in the hash map's iteration order
std::vector<MergedGroup> mergeVoxels(const VoxMap &grid) {
    std::unordered_set<uint32_t, KeyHash> visited;
    const VoxMap snapshot = grid;  // the reference iterates a copy (component_voxel_grid.hpp:114)
    std::map<std::pair<uint8_t, uint32_t>, std::vector<IBox>> byType;
    std::vector<uint32_t> expansion;
    for (const auto &kv : snapshot) {
        const uint32_t key = kv.first;
        if (visited.count(key)) continue;
        visited.emplace(key);
        const uint8_t type = kv.second.type;
        const uint32_t color = kv.second.color;
        const I3 c = voxUnkey(key);
        int mn[3] = {c.x, c.y, c.z}, mx[3] = {c.x, c.y, c.z};
        for (int axis = 0; axis < 3; ++axis)
            for (int sign = -1; sign <= 1; sign += 2) {
                while (true) {
                    int lo[3], hi[3];
                    for (int a = 0; a < 3; ++a) {
                        if (a == axis) lo[a] = hi[a] = sign > 0 ? mx[a] + 1 : mn[a] - 1;
                        else { lo[a] = mn[a]; hi[a] = mx[a]; }
                    }
                    expansion.clear();
                    bool ok = true;
                    for (int x = lo[0]; x <= hi[0] && ok; ++x)
                        for (int y = lo[1]; y <= hi[1] && ok; ++y)
                            for (int z = lo[2]; z <= hi[2]; ++z) {
                                const uint32_t k = voxKey(x, y, z);
                                const auto it = grid.find(k);
                                if (it == grid.end() || it->second.type != type || it->second.color != color || visited.count(k)) { ok = false; break; }
                                expansion.push_back(k);
                            }
                    if (!ok) break;
                    for (uint32_t k : expansion) visited.emplace(k);
                    if (sign > 0) mx[axis] += 1; else mn[axis] -= 1;
                }
            }
        IBox b;
        for (int a = 0; a < 3; ++a) { b.mn[a] = mn[a]; b.mx[a] = mx[a]; }
        byType[{type, color}].push_back(b);
    }
    std::vector<MergedGroup> out;
    for (auto &kv : byType) out.push_back({kv.first.first, kv.first.second, std::move(kv.second)});
    return out;
}

void setTerrainModel(MvTerrain &t, const IBox &bb, uint32_t color) {
    using namespace mvh;
    const float sx = float(bb.mx[0] - bb.mn[0]) * 1.0f, sy = 1.0f * 1.0f, sz = float(bb.mx[2] - bb.mn[2]) * 1.0f;
    const float px = bb.mn[0] * 1.0f + sx / 2, py = bb.mn[1] * 1.0f, pz = bb.mn[2] * 1.0f + sz / 2;
    M4 m = mul(scaling(0.5f, 0.025f, 0.5f), identity());
    m = mul(scaling(sx, sy, sz), m);
    m = mul(translation(0.0f, 0.025f, 0.0f), m);
    m = mul(translation(px, py, pz), m);
    std::memcpy(t.model, &m.c[0][0], 64);
    t.color = paletteIndex(color);
    for (int a = 0; a < 3; ++a) { t.bb[a] = bb.mn[a]; t.bb[3 + a] = bb.mx[a]; }
}

}  // namespace

static std::string lower(const std::string &name) {
    std::string n;
    for (char ch : name) n.push_back(char(std::tolower(ch)));
    return n;
}

// registered names (src/libs/scenarios/include/scenarios/init.hpp:33-56) that are implemented
int scenarioFromName(const std::string &name) {
    const std::string n = lower(name);
    if (n == "towerbuilding") return MV_SCENARIO_TOWER;
    if (n == "collect") return MV_SCENARIO_COLLECT;
    if (n == "rearrange") return MV_SCENARIO_REARRANGE;
    if (n == "sokoban") return MV_SCENARIO_SOKOBAN;
    if (n == "hexexplore") return MV_SCENARIO_HEX_EXPLORE;
    if (n == "hexmemory") return MV_SCENARIO_HEX_MEMORY;
    if (n == "empty") return MV_SCENARIO_EMPTY;
    if (n == "obstacleseasy" || n == "obstaclesmedium" || n == "obstacleshard" || n == "obstacleswalls" || n == "obstaclessteps" || n == "obstacleslava" || n == "test")
        return MV_SCENARIO_OBSTACLES;
    return -1;
}

// Scenario::initializeDefaultParameters (scenario.hpp:225-231) + ObstaclesScenario and its variants (scenario_obstacles.hpp:48-270)
FloatParams defaultFloatParams(const std::string &name) {
    const std::string n = lower(name);
    FloatParams fp{{"episodeLengthSec", 60.0f}, {"verticalLookLimitRad", 0.2f}, {"useUIRewardIndicators", 0.0f}};
    if (scenarioFromName(n) == MV_SCENARIO_SOKOBAN) fp["episodeLengthSec"] = 80.0f;  // scenario_sokoban.hpp:50-54
    if (scenarioFromName(n) == MV_SCENARIO_OBSTACLES) {
        fp["obstaclesMinNumPlatforms"] = 1; fp["obstaclesMaxNumPlatforms"] = 2; fp["obstaclesMinGap"] = 1; fp["obstaclesMaxGap"] = 2;
        fp["obstaclesMinLava"] = 1; fp["obstaclesMaxLava"] = 4; fp["obstaclesMinHeight"] = 1; fp["obstaclesMaxHeight"] = 3;
        fp["obstaclesNumAllowedMaxDifficulty"] = 1;
        if (n == "obstaclesmedium") {
            fp["obstaclesMinNumPlatforms"] = 2; fp["obstaclesMaxNumPlatforms"] = 4; fp["obstaclesMinLava"] = 2; fp["obstaclesMaxLava"] = 5;
        } else if (n == "obstacleshard") {
            fp["obstaclesMinNumPlatforms"] = 2; fp["obstaclesMaxNumPlatforms"] = 7; fp["obstaclesMinGap"] = 2; fp["obstaclesMaxGap"] = 3;
            fp["obstaclesMinLava"] = 3; fp["obstaclesMaxLava"] = 10; fp["obstaclesMinHeight"] = 2; fp["obstaclesMaxHeight"] = 4;
        } else if (n == "obstacleswalls" || n == "obstaclessteps" || n == "obstacleslava") {
            fp["obstaclesMinNumPlatforms"] = 1; fp["obstaclesMaxNumPlatforms"] = 4; fp["obstaclesMinGap"] = 1; fp["obstaclesMaxGap"] = 3;
            fp["obstaclesMinLava"] = 2; fp["obstaclesMaxLava"] = 10; fp["obstaclesMinHeight"] = 1; fp["obstaclesMaxHeight"] = 3;
        } else if (n == "test") {
            fp["obstaclesMinNumPlatforms"] = 0; fp["obstaclesMaxNumPlatforms"] = 0; fp["episodeLengthSec"] = 6.0f;
        }
    }
    return fp;
}

std::vector<std::pair<std::string, float>> defaultRewardShaping(const std::string &name) {
    const std::string n = lower(name);
    const int scenario = scenarioFromName(n);
    if (scenario == MV_SCENARIO_TOWER)  // scenario_tower_building.hpp:44-52
        return {{"teamSpirit", 0.1f}, {"towerPickedUpObject", 0.1f}, {"towerVisitedBuildingZoneWithObject", 0.1f}, {"towerBuildingReward", 1.0f}};
    if (scenario == MV_SCENARIO_COLLECT)  // scenario_collect.hpp:42-50
        return {{"collectSingleGood", 1.0f}, {"collectSingleBad", -1.0f}, {"collectAll", 5.0f}, {"collectAbyss", -0.5f}};
    if (scenario == MV_SCENARIO_OBSTACLES) {  // scenario_obstacles.hpp:37-45,201-206
        const bool oneType = n == "obstacleswalls" || n == "obstaclessteps" || n == "obstacleslava";
        return {{"obstaclesAgentAtExit", 1.0f}, {"obstaclesAllAgentsAtExit", 5.0f}, {"obstaclesExtraReward", 0.5f}, {"obstaclesAgentCarriedObjectToExit", oneType ? 1.0f : 0.0f}};
    }
    if (scenario == MV_SCENARIO_REARRANGE)  // scenario_rearrange.hpp:91-97
        return {{"rearrangeOneMoreObjectCorrectPosition", 1.0f}, {"rearrangeAllObjectsCorrectPosition", 10.0f}};
    if (scenario == MV_SCENARIO_HEX_EXPLORE) return {{"exploreSolved", 5.0f}};  // scenario_hex_explore.hpp:27-30
    if (scenario == MV_SCENARIO_HEX_MEMORY) return {{"memoryCollectGood", 1.0f}, {"memoryCollectBad", -1.0f}};  // scenario_hex_memory.hpp:43-49
    if (scenario == MV_SCENARIO_SOKOBAN)  // scenario_sokoban.hpp:41-48
        return {{"sokobanBoxOnTarget", 1.0f}, {"sokobanBoxLeavesTarget", -1.0f}, {"sokobanAllBoxesOnTarget", 10.0f}};
    return {};
}

// the shaping keys of every scenario and the reward-table slot (MV_R_*) each one fills; teamSpirit (slot 0) is every scenario's
namespace {
struct RewardSlotKey { int scenario; int slot; const char *key; };
const RewardSlotKey kRewardSlots[] = {
    {MV_SCENARIO_TOWER, MV_R_TOWER_PICKED_UP, "towerPickedUpObject"},
    {MV_SCENARIO_TOWER, MV_R_TOWER_VISITED_BZ, "towerVisitedBuildingZoneWithObject"},
    {MV_SCENARIO_TOWER, MV_R_TOWER_BUILDING, "towerBuildingReward"},
    {MV_SCENARIO_COLLECT, MV_R_COLLECT_GOOD, "collectSingleGood"},
    {MV_SCENARIO_COLLECT, MV_R_COLLECT_BAD, "collectSingleBad"},
    {MV_SCENARIO_COLLECT, MV_R_COLLECT_ALL, "collectAll"},
    {MV_SCENARIO_COLLECT, MV_R_COLLECT_ABYSS, "collectAbyss"},
    {MV_SCENARIO_OBSTACLES, MV_R_OBST_AGENT_AT_EXIT, "obstaclesAgentAtExit"},
    {MV_SCENARIO_OBSTACLES, MV_R_OBST_ALL_AT_EXIT, "obstaclesAllAgentsAtExit"},
    {MV_SCENARIO_OBSTACLES, MV_R_OBST_EXTRA, "obstaclesExtraReward"},
    {MV_SCENARIO_OBSTACLES, MV_R_OBST_CARRIED_TO_EXIT, "obstaclesAgentCarriedObjectToExit"},
    {MV_SCENARIO_HEX_EXPLORE, MV_R_EXPLORE_SOLVED, "exploreSolved"},
    {MV_SCENARIO_HEX_MEMORY, MV_R_MEMORY_GOOD, "memoryCollectGood"},
    {MV_SCENARIO_HEX_MEMORY, MV_R_MEMORY_BAD, "memoryCollectBad"},
    {MV_SCENARIO_SOKOBAN, MV_R_SOKOBAN_ON_TARGET, "sokobanBoxOnTarget"},
    {MV_SCENARIO_SOKOBAN, MV_R_SOKOBAN_LEAVES_TARGET, "sokobanBoxLeavesTarget"},
    {MV_SCENARIO_SOKOBAN, MV_R_SOKOBAN_ALL, "sokobanAllBoxesOnTarget"},
    {MV_SCENARIO_REARRANGE, MV_R_REARRANGE_ONE_MORE, "rearrangeOneMoreObjectCorrectPosition"},
    {MV_SCENARIO_REARRANGE, MV_R_REARRANGE_ALL, "rearrangeAllObjectsCorrectPosition"},
};
}  // namespace

int rewardSlot(int scenario, const std::string &key) {
    if (key == "teamSpirit") return MV_R_TEAM_SPIRIT;
    for (const RewardSlotKey &r : kRewardSlots)
        if (r.scenario == scenario && key == r.key) return r.slot;
    return -1;
}

const char *rewardKey(int scenario, int slot) {
    for (const RewardSlotKey &r : kRewardSlots)
        if (r.scenario == scenario && r.slot == slot) return r.key;
    return nullptr;
}

std::vector<uint32_t> colorTables() {
    static const uint32_t agent[7] = {C_YELLOW, C_GREEN, C_BLUE, C_ORANGE, C_VIOLET, C_VERY_DARK_GREY, C_RED};  // const.hpp:85, the step kernel's agentColors
    std::vector<uint32_t> o{22u, 7u, 14u, 14u};
    o.insert(o.end(), kPalette, kPalette + 22);
    o.insert(o.end(), agent, agent + 7);
    o.insert(o.end(), kObjectColors, kObjectColors + 14);
    o.insert(o.end(), kLayoutColors, kLayoutColors + 14);
    return o;
}

int decoCapacity(int scenario) {
    switch (scenario) {
        case MV_SCENARIO_REARRANGE: return MV_MAX_ARRANGEMENT;
        case MV_SCENARIO_SOKOBAN: return 128;       // wall / goal markers of a 10 x 10 room
        case MV_SCENARIO_HEX_EXPLORE: case MV_SCENARIO_HEX_MEMORY: return MV_MAX_DECO;  // <= 294 walls x (wall + edging + <= 4 landmarks)
        default: return 1;
    }
}

int gridCapacity(int scenario) {
    // TowerBuilding rooms are at most 29 x (6+18) x 24; Obstacles chains of up to 7 platforms (+ transitions, start, exit)
    // with the y range starting at -30; Collect: <= 41 x 41 landscape, heights <= 18, 16 cells of margin, y from -30;
    // Rearrange: 19 x (6+18) x 14 room.  None of these bounds holds every put-down: an object that ends outside the grid (beyond
    // the level's edge, sunk to y = -30 in the void, above the head-room) is found by the step kernel through its translation
    if (scenario == MV_SCENARIO_HEX_EXPLORE || scenario == MV_SCENARIO_EMPTY) return 128;  // no voxel grid
    if (scenario == MV_SCENARIO_HEX_MEMORY) return 64 * 4 * 64;  // one layer of cells over a maze of radius <= 7 * 3.5 * sqrt(3)
    // Sokoban: Boxoban rooms are 10 x 10 cells (voxel size 2), y in [-2, 6)
    const int cells = (scenario == MV_SCENARIO_TOWER || scenario == MV_SCENARIO_REARRANGE || scenario == MV_SCENARIO_SOKOBAN) ? 30 * 25 * 25 : (scenario == MV_SCENARIO_COLLECT ? 74 * 62 * 74 : 512 * 1024);
    return ((cells + 127) / 128) * 128;
}

LevelGenerator::LevelGenerator(const std::string &scenarioName, int numAgents, const FloatParams &params)
    : scenario_(scenarioFromName(scenarioName)), name_(lower(scenarioName)), numAgents_(numAgents), params_(params) {
    if (scenario_ == MV_SCENARIO_SOKOBAN) {  // SokobanScenario constructor (scenario_sokoban.cpp:39-81)
        const char *envvar = std::getenv("BOXOBAN_LEVELS");
        std::string dir = (envvar && std::strlen(envvar)) ? envvar : "~/datasets/boxoban";
        const auto tilde = dir.find('~');
        if (tilde != std::string::npos) {
            const char *home = std::getenv("HOME");
            if (!home || !std::strlen(home)) throw std::runtime_error("could not query HOME to resolve ~ in the path to the Boxoban levels");
            dir.replace(tilde, 1, home);
        }
        const std::string dirWithLevels = dir + "/unfiltered/train";  // levelSet / levelSplit (scenario_sokoban.hpp:59)
        for (int levelFileIdx = 0; levelFileIdx <= 999; ++levelFileIdx) {
            char name[16];
            std::snprintf(name, sizeof name, "%03d.txt", levelFileIdx);
            const std::string path = dirWithLevels + "/" + name;
            if (std::ifstream(path).good()) sokobanFiles_.push_back(path);
        }
        if (sokobanFiles_.empty())
            throw std::runtime_error("could not find any Boxoban levels: set BOXOBAN_LEVELS or unpack the boxoban folder (unfiltered/medium/hard) into ~/datasets");
    }
}

// the i-th static box of the level under construction (the arrays grow as needed: the reference has no bound on them)
static MvBox &staticAt(LevelOut &out, int i) {
    if (int(out.statics.size()) <= i) { out.statics.resize(size_t(i) + 1); out.staticRot.resize((size_t(i) + 1) * 2, 0.0f); }
    return out.statics[size_t(i)];
}

int LevelGenerator::generateFitting(LevelOut &out, int serial, int gridCells, int attempts) {
    for (int skipped = 0;; ++skipped) {
        try {
            generate(out, serial, gridCells);
            return skipped;
        } catch (const std::runtime_error &) {
            if (skipped + 1 >= attempts) throw;
        }
    }
}

void LevelGenerator::generate(LevelOut &out, int serial, int gridCells) {
    std::memset(&out.level, 0, sizeof(MvLevel));
    out.drawSeq.clear();
    out.deco.clear();
    out.statics.clear();
    out.staticRot.clear();
    // Env::reset: reseed the env stream from itself
    const auto sd = randRange(0, 1 << 30, rng_);
    rng_.seed((unsigned long)sd);
    episodeSeed_ = unsigned(sd);
    out.level.serial = serial;
    out.level.scenario = scenario_;
    out.level.look_limit = params_.at("verticalLookLimitRad");
    switch (scenario_) {
        case MV_SCENARIO_TOWER: generateTower(out); break;
        case MV_SCENARIO_OBSTACLES: generateObstacles(out); break;
        case MV_SCENARIO_COLLECT: generateCollect(out); break;
        case MV_SCENARIO_REARRANGE: generateRearrange(out); break;
        case MV_SCENARIO_SOKOBAN: generateSokoban(out); break;
        case MV_SCENARIO_HEX_EXPLORE: generateHexExplore(out); break;
        case MV_SCENARIO_HEX_MEMORY: generateHexMemory(out); break;
        case MV_SCENARIO_EMPTY: generateEmpty(out); break;
        default: throw std::runtime_error("unsupported scenario");
    }
    MvLevel &L = out.level;
    L.n_deco = int(out.deco.size());
    if (L.n_deco > decoCapacity(scenario_)) throw std::runtime_error("too many decorations");
    if (scenario_ == MV_SCENARIO_HEX_EXPLORE || scenario_ == MV_SCENARIO_HEX_MEMORY || scenario_ == MV_SCENARIO_EMPTY) L.n_grid_static = 0;  // no voxel grid boxes at all
    else if (scenario_ != MV_SCENARIO_REARRANGE) L.n_grid_static = L.n_static;
    if (scenario_ == MV_SCENARIO_SOKOBAN || scenario_ == MV_SCENARIO_HEX_EXPLORE || scenario_ == MV_SCENARIO_HEX_MEMORY) {  // objects sit where the generator put them
    } else
        for (int i = 0; i < L.n_obj; ++i)
            for (int a = 0; a < 3; ++a) L.obj_init[i].pos[a] = float(L.obj_init[i].voxel[a]) + 0.5f;
    assignSlots(out);
    if (L.grid_dim[0] * L.grid_dim[1] * L.grid_dim[2] > gridCells) throw std::runtime_error("level exceeds the dense grid capacity");
}

// Instance slots in the reference's draw order: mesh type major (meshIndices is a std::map<DrawableType,int>), insertion
// order minor (v4r_env_renderer.cpp:267-279).
void LevelGenerator::assignSlots(LevelOut &out) {
    MvLevel &L = out.level;
    const int A = numAgents_;
    std::vector<DrawRef> seq = out.drawSeq;
    if (seq.empty()) {
        for (int i = 0; i < L.n_static; ++i)
            if (staticAt(out, i).flags & MV_OPAQUE) seq.push_back({DrawRef::STATIC, i});
        for (int i = 0; i < L.n_terrain; ++i) seq.push_back({DrawRef::TERRAIN, i});
        for (int i = 0; i < L.n_obj; ++i) seq.push_back({DrawRef::OBJECT, i});
        seq.push_back({DrawRef::EYES, 0}); seq.push_back({DrawRef::BARS, 0}); seq.push_back({DrawRef::BODIES, 0}); seq.push_back({DrawRef::REWARDS, 0});
        L.n_static_pre = L.n_static;
    }
    L.n_opaque = 0;
    int slot = 0, terrainSeen = 0;
    for (int mesh = 0; mesh < 5; ++mesh) {
        const int first = slot;
        for (const DrawRef &d : seq) {
            switch (d.kind) {
                case DrawRef::STATIC: if (mesh == 0) { staticAt(out, d.index).flags = (staticAt(out, d.index).flags & 255) | (slot++ << 8); ++L.n_opaque; } break;
                case DrawRef::TERRAIN:  // slabs are consecutive in every scenario
                    if (mesh == 0) { if (terrainSeen++ == 0) L.slot_terrain = slot; ++slot; }
                    break;
                case DrawRef::OBJECT: if (MV_OBJ_MESH(L.obj_init[d.index].meta) == mesh) L.obj_init[d.index].meta = (L.obj_init[d.index].meta & 255) | (slot++ << 8); break;
                case DrawRef::DECO: if (out.deco[size_t(d.index)].mesh == mesh) out.deco[size_t(d.index)].slot = slot++; break;
                case DrawRef::EYES: if (mesh == 0) { L.slot_eyes = slot; slot += A; } break;
                case DrawRef::BARS: if (mesh == 0) { L.slot_bars = slot; slot += A; } break;
                case DrawRef::BODIES: if (mesh == 1) { L.slot_body = slot; slot += A; } break;
                case DrawRef::REWARDS:  // every reward object is a diamond: two cones
                    if (mesh == 3) {
                        L.slot_reward = slot;
                        for (int r = 0; r < L.n_reward; ++r) { L.reward_slot[r] = int16_t(slot); L.reward_mesh[r] = 3; L.reward_cnt[r] = 2; slot += 2; }
                    }
                    break;
                case DrawRef::REWARD_ONE:
                    if (L.reward_mesh[d.index] == mesh) { L.reward_slot[d.index] = int16_t(slot); slot += L.reward_cnt[d.index]; }
                    break;
            }
        }
        L.mesh_counts[mesh] = slot - first;
    }
    if (slot > MV_HARD_MAX_INSTANCES) throw std::runtime_error("too many drawables");
}

void LevelGenerator::generateTower(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;

    uint32_t layoutColor = randomLayoutColor(rng);
    while (layoutColor == C_DARK_GREY) layoutColor = randomLayoutColor(rng);  // != BUILDING_ZONE

    // TowerBuildingPlatform::init
    const int height = randRange(5, 7, rng);
    int length = randRange(12, 30, rng);
    int width = randRange(12, 25, rng);
    const int bzL = randRange(3, 9, rng), bzW = randRange(3, 9, rng);
    const int matL = randRange(2, 8, rng), matW = randRange(2, 8, rng);
    length = std::max(bzL + matL + 3, length);
    width = std::max(bzW + matW + 3, width);
    const int bzX = randRange(1, length - bzL - 1, rng);
    const int bzZ = randRange(1, width - bzW - 1, rng);
    const int matX = randRange(1, length - matL - 1, rng);
    const int matZ = randRange(1, width - matW - 1, rng);

    std::vector<I3> cand;
    for (int x = 1; x < length - 1; ++x)
        for (int z = 1; z < width - 1; ++z) cand.push_back({x, 2, z});
    std::shuffle(cand.begin(), cand.end(), rng);

    std::vector<I3> agentSpawn(cand.begin(), cand.begin() + std::min(A, int(cand.size())));
    const int spawnIdx = int(agentSpawn.size());
    const int maxRandomObjects = std::min(int(cand.size()) - A, 25);
    const int spawnObjects = randRange(0, std::max(1, maxRandomObjects), rng);
    std::vector<I3> objs(cand.begin() + spawnIdx, cand.begin() + spawnIdx + spawnObjects);
    for (auto &c : objs) {
        if (c.x >= matX && c.x < matX + matL && c.z >= matZ && c.z < matZ + matW) continue;
        c.y -= 1;
    }
    for (int x = matX; x < matX + matL; ++x)
        for (int z = matZ; z < matZ + matW; ++z) objs.push_back({x, 1, z});
    while (int(agentSpawn.size()) < A) agentSpawn.push_back(agentSpawn[0]);

    // generate(): floor, walls S N E W, building-zone terrain box; then (GCC argument order) drawWalls, wall colour
    const bool drawWalls = randomBool(rng);
    const uint32_t wallColor = randomLayoutColor(rng);

    VoxMap grid{100};
    fillBox(grid, {{0, 0, 0}, {length, 1, width}}, MV_SOLID | MV_OPAQUE, layoutColor);
    const uint8_t wallType = uint8_t(MV_SOLID | (drawWalls ? MV_OPAQUE : 0));
    fillBox(grid, {{0, 0, 0}, {1, height, width}}, wallType, wallColor);
    fillBox(grid, {{length - 1, 0, 0}, {length, height, width}}, wallType, wallColor);
    fillBox(grid, {{0, 0, 0}, {length, height, 1}}, wallType, wallColor);
    fillBox(grid, {{0, 0, width - 1}, {length, height, width}}, wallType, wallColor);
    const IBox bz{{bzX, 1, bzZ}, {bzX + bzL, 1, bzZ + bzW}};
    fillTerrain(grid, bz, 4);  // empty y-range: sets nothing, exactly like the reference

    // DefaultScenario::spawnAgents
    for (int i = 0; i < A; ++i) {
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = float(agentSpawn[i].x) + 0.5f, sy = float(agentSpawn[i].y) + 0.0f, sz = float(agentSpawn[i].z) + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        L.init_pos[i][0] = float(agentSpawn[i].x); L.init_pos[i][1] = float(agentSpawn[i].y); L.init_pos[i][2] = float(agentSpawn[i].z);
    }

    // addEpisodeDrawables: merged boxes (skip VOXEL_EMPTY groups), terrain slabs, movable objects
    int ns = 0;
    for (const auto &g : mergeVoxels(grid)) {
        if (g.type == 0) continue;
        for (const auto &b : g.boxes) {
            MvBox &sb = staticAt(out, ns++);
            for (int a = 0; a < 3; ++a) {
                sb.h[a] = (float(b.mx[a] - b.mn[a] + 1) / 2) * 1.0f;
                sb.c[a] = (float(b.mn[a] + b.mx[a]) / 2 + 0.5f) * 1.0f;
            }
            sb.flags = g.type;
            sb.color = paletteIndex(g.color);
        }
    }
    L.n_static = ns;
    L.n_terrain = 0;
    if (bz.mx[0] - bz.mn[0] > 0) { setTerrainModel(L.terrain[L.n_terrain], bz, C_DARK_GREY); L.terrain[L.n_terrain++].type = 4; }
    if (int(objs.size()) > MV_MAX_OBJECTS - 1) throw std::runtime_error("too many movable objects");
    L.n_obj = int(objs.size());
    L.n_movable = int(objs.size());
    L.episode_len = params_.at("episodeLengthSec") + 4.0f * float(objs.size());  // scenario_tower_building.cpp:263-266
    for (int i = 0; i < L.n_obj; ++i) {
        setStackingBox(L.obj_init[i], objs[i]);
    }
    for (int a = 0; a < 3; ++a) { L.bz_min[a] = bz.mn[a]; L.bz_max[a] = bz.mx[a]; }

    // dense grid: the room's bounding box, with head-room above the walls for stacked objects
    L.grid_org[0] = 0; L.grid_org[1] = 0; L.grid_org[2] = 0;
    L.grid_dim[0] = length; L.grid_dim[1] = height + 18; L.grid_dim[2] = width;
    fillPlanes(out, &grid);
}

// RearrangeScenario (scenario_rearrange.cpp:46-300): a 19 x 14 walled room with a target arrangement on the left pedestal
// and the same items, partly displaced, on the right one.
void LevelGenerator::generateRearrange(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    const int leftC[3] = {5, 2, 5}, rightC[3] = {13, 2, 5};
    // RearrangePlatform::init, EmptyPlatform::generate (no draws), addPlatform(..., randomBool)
    const int height = randRange(4, 7, rng), length = 19, width = 14;
    const bool drawWalls = randomBool(rng);
    VoxMap grid{100};
    fillBox(grid, {{0, 0, 0}, {length, 1, width}}, MV_SOLID | MV_OPAQUE, C_DARK_GREY);
    const uint8_t wallType = uint8_t(MV_SOLID | (drawWalls ? MV_OPAQUE : 0));
    fillBox(grid, {{0, 0, 0}, {1, height, width}}, wallType, C_DARK_GREY);
    fillBox(grid, {{length - 1, 0, 0}, {length, height, width}}, wallType, C_DARK_GREY);
    fillBox(grid, {{0, 0, 0}, {length, height, 1}}, wallType, C_DARK_GREY);
    fillBox(grid, {{0, 0, width - 1}, {length, height, width}}, wallType, C_DARK_GREY);

    // generateArrangement (:70-126)
    struct Item { int mesh; uint32_t color; I3 off; };
    static const int shapes[4] = {4, 1, 0, 2};  // Cylinder, Capsule, Box, Sphere as mesh codes (scenario_rearrange.hpp:33-35)
    auto randomItem = [&](I3 off) { Item it; it.mesh = shapes[randRange(0, 4, rng)]; it.color = randomObjectColor(rng); it.off = off; return it; };
    std::vector<Item> items;
    {
        const int arrangementSize = randRange(2, 8, rng);
        std::vector<Item> q;  // FIFO
        size_t qHead = 0;
        std::vector<I3> used;
        auto isUsed = [&](const I3 &c) { for (auto &u : used) if (u.x == c.x && u.y == c.y && u.z == c.z) return true; return false; };
        const Item first = randomItem({0, 0, 0});
        q.push_back(first); items.push_back(first); used.push_back({0, 0, 0});
        std::vector<I3> directions{{-1, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, -1}, {0, 0, 1}};
        while (qHead < q.size()) {
            const Item curr = q[qHead++];
            int maxBranches = randRange(1, int(directions.size()) + 1, rng);
            maxBranches = randRange(1, maxBranches + 1, rng);
            int numBranches = 0;
            std::shuffle(directions.begin(), directions.end(), rng);
            for (auto dir : directions) {
                const I3 no{curr.off.x + dir.x, curr.off.y + dir.y, curr.off.z + dir.z};
                const I3 below{no.x, no.y - 1, no.z};
                if (no.y >= 2 || std::abs(no.x) >= 2 || std::abs(no.z) >= 2) continue;
                if (isUsed(no)) continue;
                if (!(no.y == 0 || isUsed(below))) continue;
                const Item ni = randomItem(no);
                q.push_back(ni); items.push_back(ni); used.push_back(no);
                ++numBranches;
                if (numBranches >= maxBranches) break;
                if (int(items.size()) >= arrangementSize) break;
            }
            if (int(items.size()) >= arrangementSize) break;
        }
    }

    // DefaultScenario::spawnAgents with RearrangeScenario::agentStartingPositions (:179-200)
    std::vector<I3> agentPos(size_t(A), I3{0, 0, 0});
    for (int i = 0; i < A; ++i)
        for (int attempt = 0; attempt < 20; ++attempt) {
            const int ax = randRange(2, length - 1, rng);
            const int az = randRange(2, width - 1, rng);
            if (std::fabs(float(ax - leftC[0])) < 2 && std::fabs(float(az - leftC[2])) < 2) continue;
            if (std::fabs(float(ax - rightC[0])) < 2 && std::fabs(float(az - rightC[2])) < 2) continue;
            agentPos[size_t(i)] = {ax, 2, az};
            break;
        }
    for (int i = 0; i < A; ++i) {
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = float(agentPos[size_t(i)].x) + 0.5f, sy = float(agentPos[size_t(i)].y) + 0.0f, sz = float(agentPos[size_t(i)].z) + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        L.init_pos[i][0] = float(agentPos[size_t(i)].x); L.init_pos[i][1] = float(agentPos[size_t(i)].y); L.init_pos[i][2] = float(agentPos[size_t(i)].z);
    }

    // addEpisodeDrawables (:265-300): boxes of the voxel grid first
    int ns = 0;
    for (const auto &g : mergeVoxels(grid)) {
        if (g.type == 0) continue;
        for (const auto &b : g.boxes) {
            MvBox &sb = staticAt(out, ns);
            for (int a = 0; a < 3; ++a) {
                sb.h[a] = (float(b.mx[a] - b.mn[a] + 1) / 2) * 1.0f;
                sb.c[a] = (float(b.mn[a] + b.mx[a]) / 2 + 0.5f) * 1.0f;
            }
            sb.flags = g.type;
            sb.color = paletteIndex(g.color);
            if (g.type & MV_OPAQUE) out.drawSeq.push_back({DrawRef::STATIC, ns});
            ++ns;
        }
    }
    L.n_grid_static = ns;
    // pedestal footprints become solid voxels (placement logic only, no box): y = 1, 7 x 7 around both centres
    for (int dx = -3; dx <= 3; ++dx)
        for (int dz = -3; dz <= 3; ++dz) {
            Vox v; v.type = MV_SOLID;
            grid[voxKey(leftC[0] + dx, 1, leftC[2] + dz)] = v;
            grid[voxKey(rightC[0] + dx, 1, rightC[2] + dz)] = v;
        }

    // arrangementDrawables (:202-263): scale = scales[shape] * 0.45, collision scale (1,0.5,1) cylinder / (1,2,1) capsule
    const float objSize = 0.45f;
    auto shapeScale = [&](int mesh, float sc[3]) {
        const float b[3] = {mesh == 1 ? 0.8f : (mesh == 4 ? 0.9f : 1.0f), mesh == 1 ? 0.5f : (mesh == 4 ? 2.0f : 1.0f), mesh == 1 ? 0.8f : (mesh == 4 ? 0.9f : 1.0f)};
        for (int a = 0; a < 3; ++a) sc[a] = b[a] * objSize;
    };
    auto colScaleY = [](int mesh) { return mesh == 4 ? 0.5f : (mesh == 1 ? 2.0f : 1.0f); };
    L.n_deco = 0;
    for (const Item &it : items) {  // the target, not interactive: static colliders + drawables
        const I3 pos{it.off.x + leftC[0], it.off.y + leftC[1], it.off.z + leftC[2]};
        const float t[3] = {float(pos.x) + 0.5f, float(pos.y) + 0.5f, float(pos.z) + 0.5f};
        float sc[3];
        shapeScale(it.mesh, sc);
        MvBox &sb = staticAt(out, ns++);
        const float cs[3] = {1.0f, colScaleY(it.mesh), 1.0f};
        for (int a = 0; a < 3; ++a) { sb.c[a] = t[a] + 0.0f; sb.h[a] = std::sqrt(sc[a] * sc[a] + 0.0f * 0.0f + 0.0f * 0.0f) * cs[a]; }
        sb.flags = MV_SOLID; sb.color = 0;
        out.deco.emplace_back();
        MvDeco &d = out.deco.back();
        std::memset(d.model, 0, sizeof d.model);
        d.model[0] = sc[0]; d.model[5] = sc[1]; d.model[10] = sc[2]; d.model[12] = t[0]; d.model[13] = t[1]; d.model[14] = t[2]; d.model[15] = 1.0f;
        d.mesh = it.mesh; d.color = paletteIndex(it.color); d.slot = 0; d.pad = 0;
        out.drawSeq.push_back({DrawRef::DECO, L.n_deco});
        ++L.n_deco;
    }
    L.n_static_pre = ns;
    {   // the working copy: the first numUnmovedItems stay in place, the rest go to random free floor cells
        std::vector<I3> occupied;
        for (const Item &it : items) occupied.push_back(it.off);
        auto isOcc = [&](const I3 &c) { for (auto &u : occupied) if (u.x == c.x && u.y == c.y && u.z == c.z) return true; return false; };
        const int numUnmoved = randRange(0, int(items.size()), rng);
        int placed = 0;
        L.n_obj = 0;
        for (const Item &it : items) {
            I3 off = it.off;
            if (placed >= numUnmoved) {
                while (isOcc(off)) { const int rx = randRange(-2, 3, rng); const int rz = randRange(-2, 3, rng); off = {rx, 0, rz}; }
                occupied.push_back(off);
            }
            MvObjInit &o = L.obj_init[L.n_obj];
            o.voxel[0] = int16_t(off.x + rightC[0]); o.voxel[1] = int16_t(off.y + rightC[1]); o.voxel[2] = int16_t(off.z + rightC[2]);
            o.color = int16_t(paletteIndex(it.color));
            shapeScale(it.mesh, o.scale);
            o.meta = it.mesh | ((it.mesh == 4 ? 2 : (it.mesh == 1 ? 3 : 1)) << 3);
            out.drawSeq.push_back({DrawRef::OBJECT, L.n_obj});
            ++L.n_obj;
            ++placed;
        }
    }
    // floor slab between the pedestals and the two pedestals (addStaticCollidingBox, layout_utils.cpp:70-84)
    auto addBox = [&](float sx, float sy, float sz, float tx, float ty, float tz, uint32_t color) {
        MvBox &sb = staticAt(out, ns);
        const float sc[3] = {sx, sy, sz}, t[3] = {tx, ty, tz};
        for (int a = 0; a < 3; ++a) { sb.c[a] = t[a] + 0.0f; sb.h[a] = std::sqrt(sc[a] * sc[a] + 0.0f * 0.0f + 0.0f * 0.0f) * 1.0f; }
        sb.flags = MV_SOLID | MV_OPAQUE; sb.color = paletteIndex(color);
        out.drawSeq.push_back({DrawRef::STATIC, ns});
        ++ns;
    };
    addBox(8.35f, 0.5f, 5.65f, 9.5f + 0.0f, 0.0f + 1.0f, 7.0f + 0.0f, C_DARK_GREY);
    const float lc[3] = {float(leftC[0]), float(leftC[1]), float(leftC[2])}, rc[3] = {float(rightC[0]), float(rightC[1]), float(rightC[2])};
    addBox(3.0f, 0.5f, 3.0f, lc[0] + 0.5f, lc[1] + -0.5f, lc[2] + 0.5f, C_WHITE);
    addBox(1.5f, 0.5f, 1.5f, lc[0] + 0.5f, lc[1] + -0.45f, lc[2] + 0.5f, C_DARK_GREY);
    addBox(3.0f, 0.5f, 3.0f, lc[0] + 1.0f, lc[1] + -0.66f, lc[2] + 1.0f, C_WHITE);
    addBox(3.0f, 0.5f, 3.0f, lc[0] + 1.5f, lc[1] + -0.82f, lc[2] + 1.5f, C_WHITE);
    addBox(3.0f, 0.5f, 3.0f, rc[0] + 0.5f, rc[1] + -0.5f, rc[2] + 0.5f, C_BLUE);
    addBox(1.5f, 0.5f, 1.5f, rc[0] + 0.5f, rc[1] + -0.45f, rc[2] + 0.5f, C_DARK_GREY);
    addBox(3.0f, 0.5f, 3.0f, rc[0] + 0.0f, rc[1] + -0.66f, rc[2] + 1.0f, C_BLUE);
    addBox(3.0f, 0.5f, 3.0f, rc[0] + -0.5f, rc[1] + -0.82f, rc[2] + 1.5f, C_BLUE);
    L.n_static = ns;
    out.drawSeq.push_back({DrawRef::EYES, 0}); out.drawSeq.push_back({DrawRef::BARS, 0}); out.drawSeq.push_back({DrawRef::BODIES, 0});

    L.n_terrain = 0; L.n_reward = 0; L.n_movable = 0;
    L.episode_len = params_.at("episodeLengthSec");  // Scenario::episodeLengthSec (scenario.hpp:174-178)
    L.n_arr = int(items.size());
    for (int i = 0; i < L.n_arr; ++i) {
        L.arr[i][0] = int16_t(items[size_t(i)].mesh); L.arr[i][1] = int16_t(paletteIndex(items[size_t(i)].color));
        L.arr[i][2] = int16_t(items[size_t(i)].off.x); L.arr[i][3] = int16_t(items[size_t(i)].off.y); L.arr[i][4] = int16_t(items[size_t(i)].off.z); L.arr[i][5] = 0;
    }
    for (int a = 0; a < 3; ++a) L.work_center[a] = rightC[a];
    L.grid_org[0] = 0; L.grid_org[1] = 0; L.grid_org[2] = 0;
    L.grid_dim[0] = length; L.grid_dim[1] = height + 18; L.grid_dim[2] = width;
    fillPlanes(out, &grid);
}

// SokobanScenario (scenario_sokoban.cpp:83-295): Boxoban rooms on a voxel grid of size 2; boxes are pushed, not carried.
void LevelGenerator::generateSokoban(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    const float voxelSize = 2;
    if (sokobanLevels_.empty()) {  // reloadLevels (:83-105)
        const std::string &path = sokobanFiles_[size_t(randRange(0, int(sokobanFiles_.size()), rng))];
        std::ifstream f{path, std::ios::in | std::ios::binary};
        const std::string content((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        if (content.empty()) throw std::runtime_error("could not read the level file " + path);
        std::vector<std::string> lines;  // splitString on "\n" (strtok_r: empty lines vanish)
        for (size_t pos = 0; pos < content.size();) {
            const size_t e = content.find('\n', pos);
            const std::string tok = content.substr(pos, e == std::string::npos ? std::string::npos : e - pos);
            if (!tok.empty()) lines.push_back(tok);
            if (e == std::string::npos) break;
            pos = e + 1;
        }
        std::vector<std::string> level;
        for (int i = 0; i < int(lines.size()); ++i) {
            if (lines[size_t(i)].find(';') == 0) {
                if (i > 0) sokobanLevels_.push_back(std::move(level));  // (the file's last level is never taken, as upstream)
                level.clear();
            } else level.push_back(lines[size_t(i)]);
        }
        std::shuffle(sokobanLevels_.begin(), sokobanLevels_.end(), rng);
    }
    if (sokobanLevels_.empty()) throw std::runtime_error("Boxoban file without levels");
    const std::vector<std::string> rows = sokobanLevels_.back();
    sokobanLevels_.pop_back();

    // createLayout (:118-166)
    static const uint32_t floorColors[5] = {C_WHITE, C_VL_YELLOW, C_VL_BLUE, C_VL_ORANGE, C_DARK_GREY};
    const uint32_t floorColor = floorColors[randRange(0, 5, rng)];
    VoxMap grid{100};
    const int length = int(rows.size());
    int width = 0;
    std::vector<std::array<float, 3>> agentPos;
    std::vector<I3> boxes;
    for (int x = 0; x < length; ++x) {
        const std::string &row = rows[size_t(x)];
        width = std::max(width, int(row.size()));
        for (int z = 0; z < int(row.size()); ++z) {
            Vox fl; fl.type = MV_SOLID | MV_OPAQUE; fl.color = floorColor;
            grid[voxKey(x, 0, z)] = fl;
            const char ch = row[size_t(z)];
            if (ch == '#') {
                for (int y = 1; y <= 2; ++y) { Vox w; w.type = MV_SOLID; grid[voxKey(x, y, z)] = w; }
                grid[voxKey(x, 1, z)].terrain = 1;  // SOKO_WALL
            }
            if (ch == '@' || ch == '+')
                for (int i = 0; i < A; ++i) {
                    const float ax = float(x) + float(i % 2) * 0.5f, az = float(z) + float(i % 4 > 1) * 0.5f;
                    agentPos.push_back({ax * voxelSize, float(voxelSize + 0.3 * float(i) * voxelSize), az * voxelSize});
                }
            if (ch == '.' || ch == '+') { Vox gvx; gvx.type = 0; gvx.terrain = 2; grid[voxKey(x, 1, z)] = gvx; }  // SOKO_GOAL
            if (ch == '$' || ch == '*') boxes.push_back({x, 1, z});
        }
    }
    agentPos.resize(size_t(A), std::array<float, 3>{0, 0, 0});
    for (int i = 0; i < A; ++i) {  // DefaultScenario::spawnAgents
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = agentPos[size_t(i)][0] + 0.5f, sy = agentPos[size_t(i)][1] + 0.0f, sz = agentPos[size_t(i)][2] + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        for (int a = 0; a < 3; ++a) L.init_pos[i][a] = agentPos[size_t(i)][size_t(a)];
    }

    // addEpisodeDrawables (:229-295): merged boxes (voxel size 2), terrain markers, pushable boxes
    int ns = 0;
    for (const auto &g : mergeVoxels(grid)) {
        if (g.type == 0) continue;
        for (const auto &b : g.boxes) {
            MvBox &sb = staticAt(out, ns);
            for (int a = 0; a < 3; ++a) {
                sb.h[a] = (float(b.mx[a] - b.mn[a] + 1) / 2) * voxelSize;
                sb.c[a] = (float(b.mn[a] + b.mx[a]) / 2 + 0.5f) * voxelSize;
            }
            sb.flags = g.type;
            sb.color = paletteIndex(g.color);
            if (g.type & MV_OPAQUE) out.drawSeq.push_back({DrawRef::STATIC, ns});
            ++ns;
        }
    }
    L.n_static = ns; L.n_static_pre = ns; L.n_grid_static = ns;
    L.n_deco = 0;
    for (int x = 0; x < length; ++x)
        for (int z = 0; z < width; ++z) {
            const auto it = grid.find(voxKey(x, 1, z));
            if (it == grid.end() || it->second.terrain == 0) continue;

            const float h = it->second.terrain == 1 ? 0.35f : 0.025f;
            const float pos[3] = {voxelSize * float(x) + voxelSize / 2, voxelSize, voxelSize * float(z) + voxelSize / 2};
            mvh::M4 m = mvh::mul(mvh::scaling(1.0f, h, 1.0f), mvh::identity());
            m = mvh::mul(mvh::translation(0.0f, h, 0.0f), m);
            m = mvh::mul(mvh::translation(pos[0], pos[1], pos[2]), m);
            out.deco.emplace_back();
            MvDeco &d = out.deco.back();
            std::memcpy(d.model, &m.c[0][0], 64);
            d.mesh = 0; d.color = paletteIndex(it->second.terrain == 1 ? C_LIGHT_ORANGE : C_LIGHT_GREEN); d.slot = 0; d.pad = 0;
            out.drawSeq.push_back({DrawRef::DECO, L.n_deco});
            ++L.n_deco;
        }
    if (int(boxes.size()) > MV_MAX_OBJECTS - 1) throw std::runtime_error("too many boxes");
    L.n_obj = int(boxes.size());
    for (int i = 0; i < L.n_obj; ++i) {
        MvObjInit &o = L.obj_init[i];
        o.voxel[0] = int16_t(boxes[size_t(i)].x); o.voxel[1] = int16_t(boxes[size_t(i)].y); o.voxel[2] = int16_t(boxes[size_t(i)].z);
        o.color = int16_t(paletteIndex(C_DARK_BLUE));
        const float sc[3] = {voxelSize / 2, 0.45f, voxelSize / 2}, tr[3] = {float(boxes[size_t(i)].x) + 0.5f, float(boxes[size_t(i)].y) + 0.2f, float(boxes[size_t(i)].z) + 0.5f};
        for (int a = 0; a < 3; ++a) { o.scale[a] = sc[a] * 0.8f; o.pos[a] = tr[a] * voxelSize; }
        o.meta = 0 | (4 << 3);  // box mesh, collision scale (1.15,3,1.15) offset (0,0.6,0)
        out.drawSeq.push_back({DrawRef::OBJECT, i});
    }
    out.drawSeq.push_back({DrawRef::EYES, 0}); out.drawSeq.push_back({DrawRef::BARS, 0}); out.drawSeq.push_back({DrawRef::BODIES, 0});
    L.n_terrain = 0; L.n_reward = 0; L.n_movable = 0;
    L.episode_len = params_.at("episodeLengthSec");
    L.grid_org[0] = -2; L.grid_org[1] = -2; L.grid_org[2] = -2;
    L.grid_dim[0] = length + 4; L.grid_dim[1] = 8; L.grid_dim[2] = width + 4;
    fillPlanes(out, &grid);
}

// ---------------------------------------------------------------------------------------------------------------------
// Hexagonal mazes (src/libs/mazes: honeycombmaze.cpp, maze.cpp, kruskal.cpp; component_hexagonal_maze.cpp).  Cells are
// indexed row by row over axial coordinates (u, v); each cell keeps its remaining borders as (neighbour or -1, segment).
// A uniformly shuffled edge list + union-find carves a spanning tree (Kruskal).  Upstream seeds that shuffle from
// std::random_device, i.e. its mazes are not reproducible; here the seed is derived from the episode seed WITHOUT
// consuming the env's stream, so all other draws of the episode stay where the reference has them.
namespace {

struct HexMaze {
    struct Border { int cell; double seg[4]; };
    int n = 0, cells = 0;
    std::vector<std::vector<Border>> borders;
    std::vector<std::array<double, 2>> centers;

    int rowBegin(int u) const { return u < 0 ? -n - u + 1 : -n + 1; }
    int rowEnd(int u) const { return u < 0 ? n - 1 : n - 1 - u; }
    bool inside(int u, int v) const { return u > -n && u < n && v >= rowBegin(u) && v <= rowEnd(u); }
    int index(int u, int v) const { return u <= 0 ? ((3 * n + u) * (n + u - 1)) / 2 + v : (3 * n * (n - 1) + (4 * n - u - 1) * u) / 2 + v; }

    HexMaze(int size, unsigned seed) : n(size), cells(3 * size * (size - 1) + 1) {
        borders.resize(size_t(cells));
        centers.resize(size_t(cells));
        static const int step[6][2] = {{-1, 0}, {-1, 1}, {0, 1}, {1, 0}, {1, -1}, {0, -1}};
        const double hx = std::sqrt(3) / 2, hy = 1.5, wx = std::sqrt(3), wy = 0;
        for (int u = -n + 1; u < n; ++u)
            for (int v = rowBegin(u); v <= rowEnd(u); ++v) {
                const int me = index(u, v);
                const double cx = hx * u + wx * v, cy = hy * u + wy * v;
                centers[size_t(me)] = {cx, cy};
                for (int k = 0; k < 6; ++k) {
                    const int uu = u + step[k][0], vv = v + step[k][1];
                    const bool in = inside(uu, vv);
                    const int other = in ? index(uu, vv) : -1;
                    if (in && other > me) continue;  // the pair is recorded once, by its higher cell
                    const double a0 = (k - 2.5) * M_PI / 3, a1 = a0 + M_PI / 3;
                    Border b{other, {cx + std::cos(a0), cy + std::sin(a0), cx + std::cos(a1), cy + std::sin(a1)}};
                    borders[size_t(me)].push_back(b);
                    if (in) { b.cell = me; borders[size_t(other)].push_back(b); }
                }
            }
        // spanning tree: every tree edge loses its border on both sides
        std::vector<std::pair<int, int>> edges;
        for (int i = 0; i < cells; ++i)
            for (const Border &b : borders[size_t(i)])
                if (b.cell > i) edges.push_back({i, b.cell});
        std::mt19937 gen(seed);
        std::shuffle(edges.begin(), edges.end(), gen);
        std::vector<int> root(static_cast<size_t>(cells), 0);
        for (int i = 0; i < cells; ++i) root[size_t(i)] = i;
        auto find = [&](int x) { while (root[size_t(x)] != x) { root[size_t(x)] = root[size_t(root[size_t(x)])]; x = root[size_t(x)]; } return x; };
        auto drop = [&](int a, int b) {
            auto &l = borders[size_t(a)];
            for (size_t i = 0; i < l.size(); ++i)
                if (l[i].cell == b) { l.erase(l.begin() + long(i)); return; }
        };
        for (const auto &e : edges) {
            const int a = find(e.first), b = find(e.second);
            if (a == b) continue;
            root[size_t(a)] = b;
            drop(e.first, e.second);
            drop(e.second, e.first);
        }
    }
};

const uint32_t kAllColors[22] = {C_YELLOW, C_GREEN, C_LIGHT_GREEN, C_BLUE, C_LIGHT_BLUE, C_DARK_BLUE, C_DARK_NAVY, C_ORANGE, C_GREY, C_DARK_GREY,
                                 C_VERY_DARK_GREY, C_WHITE, C_RED, C_LIGHT_ORANGE, C_VIOLET, C_LIGHT_PINK, C_VL_YELLOW, C_VL_GREEN, C_VL_BLUE,
                                 C_VL_GREY, C_VL_VIOLET, C_VL_ORANGE};
uint32_t sampleRandomColor(Rng &rng) { return kAllColors[randRange(0, 22, rng)]; }  // const.hpp:90-94

struct HexMazeComponent {  // HexagonalMazeComponent::reset (component_hexagonal_maze.cpp:19-46)
    std::unique_ptr<HexMaze> maze;
    int size = 0;
    float scale = 3.5f, wallHeight = 1, omitProb = 0, landmarkProb = 0;
    uint32_t bottomEdging = C_WHITE, topEdging = C_WHITE;
    double xMin = 0, xMax = 0, yMin = 0, yMax = 0;
    void reset(Rng &rng, unsigned episodeSeed, int minSize, int maxSize, float omitMin, float omitMax) {
        size = randRange(minSize, maxSize, rng);
        maze = std::make_unique<HexMaze>(size, episodeSeed ^ 0x6d617a65u);
        const double xlim = std::sqrt(3) * (size - 0.5), ylim = 1.5 * size - 0.5;
        xMin = -xlim; yMin = -ylim; xMax = xlim; yMax = ylim;
        scale = 3.5f;
        wallHeight = frand(rng) * 0.55f + 0.85f;
        omitProb = frand(rng) * (omitMax - omitMin) + omitMin;
        landmarkProb = frand(rng) * 0.15f + 0.15f;
        bottomEdging = sampleRandomColor(rng);
        topEdging = sampleRandomColor(rng);
        xMin *= scale; xMax *= scale; yMin *= scale; yMax *= scale;
    }
};

void pushDeco(LevelOut &out, const mvh::M4 &m, int mesh, uint32_t color) {
    out.deco.emplace_back();
    MvDeco &d = out.deco.back();
    std::memcpy(d.model, &m.c[0][0], 64);
    d.mesh = mesh; d.color = paletteIndex(color); d.slot = 0; d.pad = 0;
    out.drawSeq.push_back({DrawRef::DECO, int(out.deco.size()) - 1});
}

// HexagonalMazeComponent::addDrawablesAndCollisions (component_hexagonal_maze.cpp:48-128): floor slab, then per remaining
// border a wall (rotated box collider + drawable), optional landmark boxes on it, and its bottom edging
void hexMazeBuild(const HexMazeComponent &hm, Rng &rng, LevelOut &out, int &ns) {
    using namespace mvh;
    MvLevel &L = out.level;
    auto colLen = [](const M4 &m, int col) { return std::sqrt(m.c[col][0] * m.c[col][0] + m.c[col][1] * m.c[col][1] + m.c[col][2] * m.c[col][2]); };
    {   // addStaticCollidingBox (layout_utils.cpp:70-84)
        const float sc[3] = {float(hm.xMax - hm.xMin), 0.0001f, float(hm.yMax - hm.yMin)};
        const float tr[3] = {float(hm.xMax + hm.xMin) / 2, 0.0f, float(hm.yMax + hm.yMin) / 2};
        const uint32_t color = randomLayoutColor(rng);
        MvBox &sb = staticAt(out, ns);
        for (int a = 0; a < 3; ++a) { sb.c[a] = tr[a] + 0.0f; sb.h[a] = std::sqrt(sc[a] * sc[a] + 0.0f * 0.0f + 0.0f * 0.0f) * 1.0f; }
        sb.flags = MV_SOLID | MV_OPAQUE; sb.color = paletteIndex(color);
        out.drawSeq.push_back({DrawRef::STATIC, ns});
        ++ns;
    }
    std::set<std::pair<int, int>> done;
    const auto &all = hm.maze->borders;
    for (int cell = 0; cell < int(all.size()); ++cell)
        for (const HexMaze::Border &b : all[size_t(cell)]) {
            std::pair<int, int> key{std::min(cell, b.cell), std::max(cell, b.cell)};
            if (b.cell != -1) {
                if (done.count(key)) continue;
                if (frand(rng) < hm.omitProb) continue;
            }
            done.insert(key);
            double x1 = b.seg[0], z1 = b.seg[1], x2 = b.seg[2], z2 = b.seg[3];
            x1 *= hm.scale; z1 *= hm.scale; x2 *= hm.scale; z2 *= hm.scale;
            const float length = 0.5f * std::sqrt(float((x1 - x2) * (x1 - x2) + (z1 - z2) * (z1 - z2)));
            const float wt[3] = {float(x1 + x2) / 2, hm.wallHeight, float(z1 + z2) / 2};
            const double dX = x1 - x2, dZ = z1 - z2;
            float rotY = float(M_PI_2);
            if (std::fabs(dX) > 1e-5f) rotY = -atanf(float(dZ / dX));
            const M4 wall = mul(translation(wt[0], wt[1], wt[2]), mul(rotationY(rotY), mul(scaling(length, hm.wallHeight, 0.15f), identity())));
            if (frand(rng) < hm.landmarkProb) {
                const float lw = 0.15f, lh = lw * length / hm.wallHeight;
                const int count = randRange(2, 5, rng);
                for (int li = 0; li < count; ++li) {
                    const float lz = frand(rng) * 1.2f + 1.5f;
                    const M4 local = mul(translation(float(li % 2 == 1) * lw * 2, float(li > 1) * lh * 2 - 0.2f, 0.0f), mul(identity(), scaling(lw, lh, lz)));
                    const uint32_t color = sampleRandomColor(rng);
                    pushDeco(out, mul(wall, local), 0, color);
                }
            }
            pushDeco(out, wall, 0, C_DARK_BLUE);
            {   // collider: centre = translation, half extents = column lengths, orientation = the normalised first column
                MvBox &sb = staticAt(out, ns);
                sb.c[0] = wall.c[3][0] + 0.0f; sb.c[1] = wall.c[3][1] + 0.0f; sb.c[2] = wall.c[3][2] + 0.0f;
                for (int a = 0; a < 3; ++a) sb.h[a] = colLen(wall, a) * 1.0f;
                sb.flags = MV_SOLID | MV_ROTATED; sb.color = 0;
                const float lenInv = 1.0f / sb.h[0];  // what Bullet is handed: Matrix4::rotation() = column * (1 / length)
                out.staticRot[size_t(ns) * 2] = wall.c[0][0] * lenInv;
                out.staticRot[size_t(ns) * 2 + 1] = wall.c[0][2] * lenInv;
                ++ns;
            }
            const float es[3] = {length * 1.02f, hm.wallHeight * 0.12f, 0.2f};
            pushDeco(out, mul(translation(wt[0], es[1], wt[2]), mul(rotationY(rotY), mul(scaling(es[0], es[1], es[2]), identity()))), 0, hm.bottomEdging);
        }
}

mvh::M4 coneBottomLocal() {  // addDiamond's lower half: rotateXLocal(180 deg) then translate(0,-1,0) (layout_utils.cpp:117-119)
    using namespace mvh;
    const float ang = 180.0f * 3.14159265358979323846f / 180.0f;
    M4 rx = identity();
    const float s = crsin(ang), c = crcos(ang);
    rx.c[1][1] = c; rx.c[1][2] = s; rx.c[2][1] = -s; rx.c[2][2] = c;
    return mul(translation(0.0f, -1.0f, 0.0f), mul(identity(), rx));
}

}  // namespace

// HexExploreScenario (scenario_hex_explore.cpp:22-108): find the diamond hidden in the maze
void LevelGenerator::generateHexExplore(LevelOut &out) {
    using namespace mvh;
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    HexMazeComponent hm;
    hm.reset(rng, episodeSeed_, 2, 8, 0.1f, 0.4f);
    const auto &centers = hm.maze->centers;
    const int rewardCell = randRange(0, int(centers.size()), rng);
    const float rc[3] = {float(centers[size_t(rewardCell)][0]) * hm.scale, 0.0f, float(centers[size_t(rewardCell)][1]) * hm.scale};
    // agentStartingPositions (:63-99): the first shuffled cell farther from the diamond than size * scale, agents on a unit circle
    std::vector<int> order(centers.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = int(i);
    std::shuffle(order.begin(), order.end(), rng);
    std::vector<std::array<float, 3>> spawn;
    float farthest = 0;
    for (int cell : order) {
        const float sp[3] = {float(centers[size_t(cell)][0]) * hm.scale, float(0.1), float(centers[size_t(cell)][1]) * hm.scale};
        const float dx = rc[0] - sp[0], dy = rc[1] - sp[1], dz = rc[2] - sp[2];
        const float distance = std::sqrt(dx * dx + dy * dy + dz * dz);
        const float rotation = float(2 * M_PI / A);
        if (distance > farthest) {
            spawn.clear();
            for (int i = 0; i < A; ++i) spawn.push_back({sp[0] + sinf(float(i) * rotation), sp[1] + 0.0f, sp[2] + cosf(float(i) * rotation)});
            farthest = distance;
        }
        if (distance > float(hm.size) * hm.scale) break;
    }
    if (spawn.empty()) spawn.assign(size_t(A), std::array<float, 3>{0, 1, 0});
    for (int i = 0; i < A; ++i) {  // DefaultScenario::spawnAgents
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = spawn[size_t(i)][0] + 0.5f, sy = spawn[size_t(i)][1] + 0.0f, sz = spawn[size_t(i)][2] + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        for (int a = 0; a < 3; ++a) L.init_pos[i][a] = spawn[size_t(i)][size_t(a)];
    }
    int ns = 0;
    hexMazeBuild(hm, rng, out, ns);
    L.n_static = ns; L.n_static_pre = ns; L.n_grid_static = 0;
    // the diamond (addDiamond, layout_utils.cpp:114-126)
    const float sc = 1.9f;
    const M4 root = mul(translation(rc[0] + 0.0f, rc[1] + 1.2f, rc[2] + 0.0f), mul(scaling(0.17f * sc, 0.35f * sc, 0.17f * sc), identity()));
    const M4 bottom = coneBottomLocal();
    std::memcpy(L.cone_bottom_local, &bottom.c[0][0], 64);
    L.n_reward = 1; L.n_positive = 0;
    std::memcpy(L.reward_root[0], &root.c[0][0], 64);
    L.reward_voxel[0][0] = L.reward_voxel[0][1] = L.reward_voxel[0][2] = 0; L.reward_voxel[0][3] = int16_t(paletteIndex(C_VIOLET));
    L.goal[0] = rc[0]; L.goal[1] = rc[1]; L.goal[2] = rc[2];
    out.drawSeq.push_back({DrawRef::EYES, 0}); out.drawSeq.push_back({DrawRef::BARS, 0}); out.drawSeq.push_back({DrawRef::BODIES, 0});
    out.drawSeq.push_back({DrawRef::REWARDS, 0});
    L.n_terrain = 0; L.n_obj = 0; L.n_movable = 0;
    L.episode_len = params_.at("episodeLengthSec");
    L.grid_org[0] = 0; L.grid_org[1] = 0; L.grid_org[2] = 0;
    L.grid_dim[0] = 1; L.grid_dim[1] = 1; L.grid_dim[2] = 1;
    out.solid.assign(1, 0u); out.exitBits.assign(1, 0u); out.lavaBits.assign(1, 0u);
}

// EmptyScenario (scenario_empty.cpp:15-30): every agent at (1,1,1), one static colliding box, no rules, no rewards
void LevelGenerator::generateEmpty(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    for (int i = 0; i < A; ++i) {  // DefaultScenario::spawnAgents
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = 1.0f + 0.5f, sy = 1.0f + 0.0f, sz = 1.0f + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        for (int a = 0; a < 3; ++a) L.init_pos[i][a] = 1.0f;
    }
    {   // addStaticCollidingBox(drawables, envState, {10, 1, 10}, {5, 0, 5}, ColorRgb::BLUE) (layout_utils.cpp:70-84)
        const float sc[3] = {10.0f, 1.0f, 10.0f}, tr[3] = {5.0f, 0.0f, 5.0f};
        MvBox &sb = staticAt(out, 0);
        for (int a = 0; a < 3; ++a) { sb.c[a] = tr[a] + 0.0f; sb.h[a] = std::sqrt(sc[a] * sc[a] + 0.0f * 0.0f + 0.0f * 0.0f) * 1.0f; }
        sb.flags = MV_SOLID | MV_OPAQUE; sb.color = paletteIndex(C_BLUE);
        out.drawSeq.push_back({DrawRef::STATIC, 0});
    }
    out.drawSeq.push_back({DrawRef::EYES, 0}); out.drawSeq.push_back({DrawRef::BARS, 0}); out.drawSeq.push_back({DrawRef::BODIES, 0});
    L.n_static = 1; L.n_static_pre = 1; L.n_grid_static = 0;
    L.n_terrain = 0; L.n_obj = 0; L.n_movable = 0; L.n_reward = 0; L.n_positive = 0;
    L.episode_len = params_.at("episodeLengthSec");  // Scenario::episodeLengthSec (scenario.hpp:174-178)
    L.grid_org[0] = 0; L.grid_org[1] = 0; L.grid_org[2] = 0;
    L.grid_dim[0] = 1; L.grid_dim[1] = 1; L.grid_dim[2] = 1;
    out.solid.assign(1, 0u); out.exitBits.assign(1, 0u); out.lavaBits.assign(1, 0u);
}

// HexMemoryScenario (scenario_hex_memory.cpp:19-217): a landmark object in the central cell shows which objects to collect
void LevelGenerator::generateHexMemory(LevelOut &out) {
    using namespace mvh;
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    HexMazeComponent hm;
    hm.reset(rng, episodeSeed_, 2, 8, 0.1f, 0.95f);
    const auto &centers = hm.maze->centers;
    const int numCells = int(centers.size());
    float minDist = 1e9f;
    int centerCell = 0;
    for (int c = 0; c < numCells; ++c) {
        const double d = std::sqrt(centers[size_t(c)][0] * centers[size_t(c)][0] + centers[size_t(c)][1] * centers[size_t(c)][1]);
        if (d < minDist) { centerCell = c; minDist = float(d); }
    }
    const float landmark[3] = {float(centers[size_t(centerCell)][0] * hm.scale), 1.0f, float(centers[size_t(centerCell)][1] * hm.scale)};
    std::vector<std::array<float, 3>> coords;
    for (int c = 0; c < numCells; ++c) {
        if (c == centerCell) continue;
        // Vector3(frand - 0.5f, 0, frand - 0.5f): GCC evaluates call arguments right to left, z is drawn first
        const float oz = frand(rng) - 0.5f;
        const float ox = frand(rng) - 0.5f;
        const float cx = float(centers[size_t(c)][0]) + ox, cy = 0.5f + 0.0f, cz = float(centers[size_t(c)][1]) + oz;
        coords.push_back({cx * hm.scale, cy, cz * hm.scale});
    }
    std::shuffle(coords.begin(), coords.end(), rng);
    const float fraction = frand(rng) * 0.25f + 0.2f;
    const long nGood = std::lround(ceilf(fraction * coords.size())), nBadWanted = nGood;
    const long nBad = long(coords.size()) >= nGood + nBadWanted ? nBadWanted : 0;
    // agents: evenly spaced on a circle of radius 1.5 around the origin, heading = their angle, no draws (:121-153)
    const float rot = float(2 * M_PI / A);
    for (int i = 0; i < A; ++i) {
        const float p[3] = {sinf(rot * float(i)) * 1.5f, float(0.3) * 1.5f, cosf(rot * float(i)) * 1.5f};
        spawnBasis(rot * i, L.spawn_basis[i]);
        const float sx = p[0] + 0.5f, sy = p[1] + 0.0f, sz = p[2] + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        for (int a = 0; a < 3; ++a) L.init_pos[i][a] = p[a];
    }
    // addEpisodeDrawables (:156-217)
    enum { PILLAR, DIAMOND, SPHERE };
    uint32_t goodColor = randomObjectColor(rng), badColor = goodColor;
    int goodShape = randRange(0, 3, rng), badShape = goodShape;
    while (badColor == goodColor && badShape == goodShape) { badColor = randomObjectColor(rng); badShape = randRange(0, 3, rng); }
    int ns = 0;
    hexMazeBuild(hm, rng, out, ns);
    L.n_static = ns; L.n_static_pre = ns; L.n_grid_static = 0;
    const M4 bottom = coneBottomLocal();
    std::memcpy(L.cone_bottom_local, &bottom.c[0][0], 64);
    auto shapeScale = [](int shape, float sc[3]) {
        if (shape == SPHERE) { sc[0] = sc[1] = sc[2] = 0.75f; }
        else if (shape == PILLAR) { sc[0] = 0.5f; sc[1] = 2.0f; sc[2] = 0.5f; }
        else { sc[0] = 0.17f * float(2.2); sc[1] = 0.45f * float(2.2); sc[2] = 0.17f * float(2.2); }
    };
    auto shapeShift = [](int shape, float sh[3]) {
        sh[0] = 0.5f; sh[2] = 0.5f;
        sh[1] = shape == SPHERE ? 0.1f : (shape == PILLAR ? 0.05f : 0.6f);
    };
    // one object: root = T(loc) * S(scale); diamonds add the shared lower-cone local, pillars two caps re-parented keeping their pose
    auto build = [&](int shape, const float loc[3], const float sc[3], M4 &root, M4 child[2], int &mesh, int &cnt) {
        root = mul(translation(loc[0], loc[1], loc[2]), mul(scaling(sc[0], sc[1], sc[2]), identity()));
        if (shape == SPHERE) { mesh = 2; cnt = 1; }
        else if (shape == DIAMOND) { mesh = 3; cnt = 2; child[0] = bottom; }
        else {
            mesh = 4; cnt = 3;
            const float capScale[3] = {sc[0] * 1.2f, 0.15f, sc[2] * 1.2f}, capT[3] = {0.0f * sc[0], 0.47f * sc[1], 0.0f * sc[2]};
            const M4 inv = inverted(root);
            for (int k = 0; k < 2; ++k) {
                const float sgn = k == 0 ? 1.0f : -1.0f;
                const float t[3] = {k == 0 ? loc[0] + capT[0] : loc[0] - capT[0], k == 0 ? loc[1] + capT[1] : loc[1] - capT[1], k == 0 ? loc[2] + capT[2] : loc[2] - capT[2]};
                (void)sgn;
                child[k] = mul(inv, mul(translation(t[0], t[1], t[2]), mul(scaling(capScale[0], capScale[1], capScale[2]), identity())));
            }
        }
    };
    {   // the landmark: static
        float sc[3], sh[3];
        shapeScale(goodShape, sc); shapeShift(goodShape, sh);
        const float loc[3] = {landmark[0] + sh[0], landmark[1] + sh[1], landmark[2] + sh[2]};
        M4 root, child[2]; int mesh, cnt;
        build(goodShape, loc, sc, root, child, mesh, cnt);
        pushDeco(out, root, mesh, goodColor);
        for (int k = 1; k < cnt; ++k) pushDeco(out, mul(root, child[k - 1]), mesh, goodColor);
    }
    const float objScale = float(0.6);
    if (nGood + nBad > MV_MAX_REWARD) throw std::runtime_error("too many collectable objects");
    L.n_reward = int(nGood + nBad); L.n_positive = int(nGood);
    for (int r = 0; r < L.n_reward; ++r) {
        const bool good = r < nGood;
        const int shape = good ? goodShape : badShape;
        const auto &c = coords[size_t(r)];
        float sc[3], sh[3];
        shapeScale(shape, sc); shapeShift(shape, sh);
        const float loc[3] = {c[0] + sh[0] * objScale, c[1] + sh[1] * objScale, c[2] + sh[2] * objScale};
        const float scs[3] = {sc[0] * objScale, sc[1] * objScale, sc[2] * objScale};
        M4 root, child[2]; int mesh, cnt;
        build(shape, loc, scs, root, child, mesh, cnt);
        std::memcpy(L.reward_root[r], &root.c[0][0], 64);
        if (mesh == 4) { std::memcpy(L.reward_child[r][0], &child[0].c[0][0], 64); std::memcpy(L.reward_child[r][1], &child[1].c[0][0], 64); }
        L.reward_mesh[r] = int8_t(mesh); L.reward_cnt[r] = int8_t(cnt);
        if (good) L.reward_good[r >> 5] |= 1u << (r & 31);
        L.reward_voxel[r][0] = int16_t(std::lround(std::floor(c[0]))); L.reward_voxel[r][1] = int16_t(std::lround(std::floor(c[1]))); L.reward_voxel[r][2] = int16_t(std::lround(std::floor(c[2])));
        L.reward_voxel[r][3] = int16_t(paletteIndex(good ? goodColor : badColor));
        out.drawSeq.push_back({DrawRef::REWARD_ONE, r});
    }
    out.drawSeq.push_back({DrawRef::EYES, 0}); out.drawSeq.push_back({DrawRef::BARS, 0}); out.drawSeq.push_back({DrawRef::BODIES, 0});
    L.n_terrain = 0; L.n_obj = 0; L.n_movable = 0;
    L.episode_len = params_.at("episodeLengthSec") + 3.0f * float(nGood);  // scenario_hex_memory.hpp:51-55
    L.grid_org[0] = 0; L.grid_org[1] = 0; L.grid_org[2] = 0;
    L.grid_dim[0] = 1; L.grid_dim[1] = 1; L.grid_dim[2] = 1;
    out.solid.assign(1, 0u); out.exitBits.assign(1, 0u); out.lavaBits.assign(1, 0u);
}

// three bit planes over the dense grid: solid, exit terrain, lava terrain
void LevelGenerator::fillPlanes(LevelOut &out, const void *gridPtr) {
    const VoxMap &grid = *static_cast<const VoxMap *>(gridPtr);
    const MvLevel &L = out.level;
    const int cells = L.grid_dim[0] * L.grid_dim[1] * L.grid_dim[2];
    const size_t words = size_t(cells + 31) / 32;
    out.solid.assign(words, 0u); out.exitBits.assign(words, 0u); out.lavaBits.assign(words, 0u);
    for (const auto &kv : grid) {
        const I3 c = voxUnkey(kv.first);
        const int gx = c.x - L.grid_org[0], gy = c.y - L.grid_org[1], gz = c.z - L.grid_org[2];
        if (gx < 0 || gy < 0 || gz < 0 || gx >= L.grid_dim[0] || gy >= L.grid_dim[1] || gz >= L.grid_dim[2]) throw std::runtime_error("voxel outside the dense grid");
        const int idx = (gx * L.grid_dim[1] + gy) * L.grid_dim[2] + gz;
        if (kv.second.type & MV_SOLID) out.solid[size_t(idx >> 5)] |= 1u << (idx & 31);
        if (kv.second.terrain & 1) out.exitBits[size_t(idx >> 5)] |= 1u << (idx & 31);
        if (kv.second.terrain & 2) out.lavaBits[size_t(idx >> 5)] |= 1u << (idx & 31);
    }
}

// ---------------------------------------------------------------------------------------------------- Collect
// scenario_collect.cpp:35-143 (createLandscape), :185-212 (reward diamonds); terrain from siv::PerlinNoise
// (src/libs/util/include/util/perlin_noise.hpp: Ken Perlin's improved noise in double precision, permutation = std::shuffle
// of 0..255 with std::default_random_engine(seed))
namespace {

class Perlin {
public:
    explicit Perlin(std::uint32_t seed) {
        for (size_t i = 0; i < 256; ++i) p[i] = static_cast<std::uint8_t>(i);
        std::shuffle(std::begin(p), std::begin(p) + 256, std::default_random_engine(seed));
        for (size_t i = 0; i < 256; ++i) p[256 + i] = p[i];
    }
    double octaves01(double x, double y, int octaves) const {  // accumulatedOctaveNoise2D_0_1
        double result = 0, amp = 1;
        for (int i = 0; i < octaves; ++i) {
            result += noise(x, y, 0) * amp;
            x *= 2; y *= 2; amp /= 2;
        }
        return std::clamp<double>(result * 0.5 + 0.5, 0, 1);
    }

private:
    static double fade(double t) { return t * t * t * (t * (t * 6 - 15) + 10); }
    static double lerp(double t, double a, double b) { return a + t * (b - a); }
    static double grad(std::uint8_t hash, double x, double y, double z) {
        const std::uint8_t h = hash & 15;
        const double u = h < 8 ? x : y;
        const double v = h < 4 ? y : h == 12 || h == 14 ? x : z;
        return ((h & 1) == 0 ? u : -u) + ((h & 2) == 0 ? v : -v);
    }
    double noise(double x, double y, double z) const {
        const int X = static_cast<int>(std::floor(x)) & 255, Y = static_cast<int>(std::floor(y)) & 255, Z = static_cast<int>(std::floor(z)) & 255;
        x -= std::floor(x); y -= std::floor(y); z -= std::floor(z);
        const double u = fade(x), v = fade(y), w = fade(z);
        const int A = p[X] + Y, AA = p[A] + Z, AB = p[A + 1] + Z, B = p[X + 1] + Y, BA = p[B] + Z, BB = p[B + 1] + Z;
        return lerp(w, lerp(v, lerp(u, grad(p[AA], x, y, z), grad(p[BA], x - 1, y, z)), lerp(u, grad(p[AB], x, y - 1, z), grad(p[BB], x - 1, y - 1, z))),
                    lerp(v, lerp(u, grad(p[AA + 1], x, y, z - 1), grad(p[BA + 1], x - 1, y, z - 1)),
                         lerp(u, grad(p[AB + 1], x, y - 1, z - 1), grad(p[BB + 1], x - 1, y - 1, z - 1))));
    }
    std::uint8_t p[512];
};

}  // namespace

void LevelGenerator::generateCollect(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    static const uint32_t landscapeColors[7] = {C_WHITE, C_VL_GREEN, C_VL_BLUE, C_VL_GREY, C_VL_ORANGE, C_GREY, C_DARK_GREY};
    static const uint32_t floorColors[3] = {C_GREY, C_DARK_GREY, C_DARK_GREY};
    const uint32_t landscapeColor = landscapeColors[randRange(0, 7, rng)];
    const uint32_t floorColor = floorColors[randRange(0, 3, rng)];
    constexpr int maxWidth = 42, maxLength = maxWidth;
    const int width = randRange(8, maxWidth, rng);
    const int length = randRange(8, maxWidth, rng);
    std::vector<int> spawnHeight(size_t(length * width), 1);
    const double frequency = double(randRange(1, 100, rng)) / 10.0;
    const int octaves = randRange(1, 10, rng);
    const std::uint32_t seed = std::uint32_t(randRange(0, 1000000000, rng));
    const Perlin perlin(seed);
    const double fx = maxLength / frequency, fz = maxWidth / frequency;
    const int intensity = randRange(5, 18, rng);
    const float groundLevel = frand(rng) * 0.5f + 0.2f;

    VoxMap grid{100};
    auto setVox = [&](int x, int y, int z, uint32_t color) { Vox v; v.type = MV_SOLID | MV_OPAQUE; v.terrain = 0; v.color = color; grid[voxKey(x, y, z)] = v; };
    for (int x = 1; x < length - 1; ++x)
        for (int z = 1; z < width - 1; ++z) {
            const double noise = perlin.octaves01(x / fx, z / fz, octaves);
            const double yCoord = intensity * (noise - groundLevel);
            if (yCoord >= 1) {
                const int yr = int(lround(yCoord));
                for (int y = yr; y >= 1; --y) setVox(x, y, z, landscapeColor);
                spawnHeight[size_t(x * width + z)] = yr + 1;
            }
        }
    for (int x = 0; x < length; ++x)
        for (int z = 0; z < width; ++z) setVox(x, 0, z, floorColor);

    std::vector<I3> spawn;
    for (int x = 1; x < length - 1; ++x)
        for (int z = 1; z < width - 1; ++z) spawn.push_back({x, spawnHeight[size_t(x * width + z)], z});
    std::shuffle(spawn.begin(), spawn.end(), rng);
    int offset = 0;
    if (int(spawn.size()) < A + 1) throw std::runtime_error("landscape too small for the agents");
    std::vector<I3> agentSpawn(spawn.begin(), spawn.begin() + A);
    offset += A;
    int numRewards = randRange(1, int(lround(0.05 * width * length)) + 2, rng);
    numRewards = std::min(numRewards, int(spawn.size()) - offset);
    const int numRandom = std::max(numRewards / 2, 1);
    std::vector<I3> rewards(spawn.begin() + offset, spawn.begin() + offset + numRandom);
    offset += numRandom;
    // same (unstable) std::sort call on the same data as the reference: equal-height order is libstdc++'s introsort order
    std::sort(spawn.begin() + offset, spawn.end(), [&](const I3 &a, const I3 &b) {
        const int ha = spawnHeight[size_t(a.x * width + a.z)], hb = spawnHeight[size_t(b.x * width + b.z)];
        if (ha != hb) return ha > hb;
        else return false;
    });
    rewards.insert(rewards.end(), spawn.begin() + offset, spawn.begin() + offset + (numRewards - numRandom));
    offset += numRewards - numRandom;
    std::shuffle(spawn.begin() + offset, spawn.end(), rng);
    const int objectsMin = std::max(3, int(length * width * 0.04));
    const int objectsMax = std::min(objectsMin + 1, int(lround(0.07 * width * length)) + 2);
    const int numObjects = std::min(randRange(objectsMin, objectsMax, rng), int(spawn.size()) - offset);
    std::vector<I3> objs;
    if (offset + numObjects < int(spawn.size())) objs.assign(spawn.begin() + offset, spawn.begin() + offset + numObjects);

    // DefaultScenario::spawnAgents
    for (int i = 0; i < A; ++i) {
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = float(agentSpawn[size_t(i)].x) + 0.5f, sy = float(agentSpawn[size_t(i)].y) + 0.0f, sz = float(agentSpawn[size_t(i)].z) + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        L.init_pos[i][0] = float(agentSpawn[size_t(i)].x); L.init_pos[i][1] = float(agentSpawn[size_t(i)].y); L.init_pos[i][2] = float(agentSpawn[size_t(i)].z);
    }

    int ns = 0;
    for (const auto &g : mergeVoxels(grid)) {
        if (g.type == 0) continue;
        for (const auto &b : g.boxes) {
            MvBox &sb = staticAt(out, ns++);
            for (int a = 0; a < 3; ++a) {
                sb.h[a] = (float(b.mx[a] - b.mn[a] + 1) / 2) * 1.0f;
                sb.c[a] = (float(b.mn[a] + b.mx[a]) / 2 + 0.5f) * 1.0f;
            }
            sb.flags = g.type;
            sb.color = paletteIndex(g.color);
        }
    }
    L.n_static = ns;
    L.n_terrain = 0;
    if (int(objs.size()) > MV_MAX_OBJECTS - 1) throw std::runtime_error("too many movable objects");
    L.n_obj = int(objs.size());
    for (int i = 0; i < L.n_obj; ++i) {
        setStackingBox(L.obj_init[i], objs[size_t(i)]);
    }
    if (int(rewards.size()) > MV_MAX_REWARD) throw std::runtime_error("too many reward objects");
    L.n_reward = int(rewards.size());
    L.n_positive = 0;
    {
        using namespace mvh;
        const float ang = 180.0f * 3.14159265358979323846f / 180.0f;
        M4 rx = identity();
        const float s = crsin(ang), c = crcos(ang);
        rx.c[1][1] = c; rx.c[1][2] = s; rx.c[2][1] = -s; rx.c[2][2] = c;
        const M4 bottom = mul(translation(0.0f, -1.0f, 0.0f), mul(identity(), rx));
        std::memcpy(L.cone_bottom_local, &bottom.c[0][0], 64);
        for (int i = 0; i < L.n_reward; ++i) {
            const I3 r = rewards[size_t(i)];
            const bool good = frand(rng) > 0.3f;  // drawn in addEpisodeDrawables, i.e. after the agents' yaw draws
            if (good) ++L.n_positive;
            L.reward_voxel[i][0] = int16_t(r.x); L.reward_voxel[i][1] = int16_t(r.y); L.reward_voxel[i][2] = int16_t(r.z);
            L.reward_voxel[i][3] = int16_t(paletteIndex(good ? C_GREEN : C_RED));
            const M4 root = mul(translation(float(r.x) + 0.5f, float(r.y) + 0.8f, float(r.z) + 0.5f), mul(scaling(0.17f, 0.45f, 0.17f), identity()));
            std::memcpy(L.reward_root[i], &root.c[0][0], 64);
        }
    }
    L.episode_len = params_.at("episodeLengthSec") + 2.0f * rewards.size();  // scenario_collect.hpp:52-56
    L.n_movable = 0;

    int maxY = 0;
    for (const auto &kv : grid) maxY = std::max(maxY, voxUnkey(kv.first).y);
    for (auto &c : objs) maxY = std::max(maxY, c.y);
    for (auto &c : rewards) maxY = std::max(maxY, c.y);
    // margin and y from -30: objects put down near the landscape's edge, or sunk to y = -30 off it, stay in the grid; those
    // beyond it are exact too (the step kernel's objAt), the margin only keeps them on the grid's fast path
    L.grid_org[0] = -16; L.grid_org[1] = -30; L.grid_org[2] = -16;
    L.grid_dim[0] = length + 32; L.grid_dim[1] = maxY + 30 + 1 + 12; L.grid_dim[2] = width + 32;
    fillPlanes(out, &grid);
}

// ---------------------------------------------------------------------------------------------------- Obstacles
// Platforms live in integer frames: origin + quarter turns about Y.  The reference pushes integer boxes through float
// scene-graph matrices (90 degree turns, integer translations) and recovers integers with lround / floor(x+0.5)
// (platforms.hpp:113-134,153-163,268-276); the accumulated float error over a chain is << 0.5, so exact integer frames
// give the same voxels (SURVEY.md Appendix C), and tests/test_cpu.py checks that against the oracle's float scene graph.
namespace {

struct Frame {
    int o[3] = {0, 0, 0};
    int r = 0;  // quarter turns, Magnum rotationY(+90 deg): x' = z, z' = -x
    void rot(int x, int z, int &xo, int &zo) const {
        switch (r & 3) {
            case 0: xo = x; zo = z; break;
            case 1: xo = z; zo = -x; break;
            case 2: xo = -x; zo = -z; break;
            default: xo = -z; zo = x; break;
        }
    }
    I3 apply(int x, int y, int z) const { int xr, zr; rot(x, z, xr, zr); return {xr + o[0], y + o[1], zr + o[2]}; }
    // voxel of the transformed cell centre (x+0.5, y+0.5, z+0.5): done on doubled coordinates, exact
    I3 applyCentre(int x, int y, int z) const {
        int xr, zr;
        rot(2 * x + 1, 2 * z + 1, xr, zr);
        const int X = xr + 2 * o[0], Z = zr + 2 * o[2];
        return {(X - 1) / 2 + ((X - 1) % 2 != 0 && X - 1 < 0 ? -1 : 0), y + o[1], (Z - 1) / 2 + ((Z - 1) % 2 != 0 && Z - 1 < 0 ? -1 : 0)};
    }
    Frame child(int tx, int ty, int tz, int turns) const {  // this * (RotY(turns) then translateLocal(t)) == rotation first, then t in the rotated frame
        Frame c;
        c.r = (r + turns) & 3;
        // origin of the child = this(RotY(turns) * t)
        Frame local;
        local.r = turns & 3;
        int xr, zr;
        local.rot(tx, tz, xr, zr);
        const I3 p = apply(xr, ty, zr);
        c.o[0] = p.x; c.o[1] = p.y; c.o[2] = p.z;
        return c;
    }
};

enum { PT_EMPTY, PT_WALL, PT_LAVA, PT_STEP, PT_GAP, PT_START, PT_EXIT, PT_TRANSITION };
enum { W_SOUTH = 1, W_NORTH = 2, W_WEST = 4, W_EAST = 8 };

struct Plat {
    int type = PT_EMPTY, walls = 0;
    int length = 0, height = 0, width = -1;
    Frame parent, root, anchor;
    std::vector<IBox> layout, wallBoxes;            // local, max exclusive
    std::vector<std::pair<int, IBox>> terrain;      // (terrain type, local box), std::map order = type order
    std::map<std::pair<int, int>, int> occupancy;
    int wallHeight = 0, lavaLength = 0, stepHeight = 0, gap = 0, gapX = 0;
    int anchorLocal[3] = {0, 0, 0};  // nextPlatformAnchor relative to the root

    IBox world(const IBox &b) const {  // MagnumAABB::boundingBox: transform both corners, sort
        const I3 a = root.apply(b.mn[0], b.mn[1], b.mn[2]), c = root.apply(b.mx[0], b.mx[1], b.mx[2]);
        IBox o;
        o.mn[0] = std::min(a.x, c.x); o.mx[0] = std::max(a.x, c.x);
        o.mn[1] = std::min(a.y, c.y); o.mx[1] = std::max(a.y, c.y);
        o.mn[2] = std::min(a.z, c.z); o.mx[2] = std::max(a.z, c.z);
        return o;
    }
    void addFloor() { layout.push_back({{0, 0, 0}, {length, 1, width}}); anchorLocal[0] = length; anchorLocal[1] = 0; anchorLocal[2] = 0; }
    void addWalls() {
        if (walls & W_SOUTH) wallBoxes.push_back({{0, 0, 0}, {1, height, width}});
        if (walls & W_NORTH) wallBoxes.push_back({{length - 1, 0, 0}, {length, height, width}});
        if (walls & W_EAST) wallBoxes.push_back({{0, 0, 0}, {length, height, 1}});
        if (walls & W_WEST) wallBoxes.push_back({{0, 0, width - 1}, {length, height, width}});
    }
    IBox outer() const {  // Platform::platformBoundingBox
        IBox o{};
        bool have = false;
        auto add = [&](const IBox &w) {
            if (!have) { o = w; have = true; return; }
            for (int a = 0; a < 3; ++a) { o.mn[a] = std::min(o.mn[a], std::min(w.mn[a], w.mx[a])); o.mx[a] = std::max(o.mx[a], std::max(w.mn[a], w.mx[a])); }
        };
        if (!layout.empty()) add(world(layout.front())); else if (!wallBoxes.empty()) add(world(wallBoxes.front()));
        for (auto &b : layout) add(world(b));
        for (auto &b : wallBoxes) add(world(b));
        return o;
    }
};

int P(const FloatParams &p, const char *k) { return int(lroundf(p.at(k))); }
int tri(int n) { return n * (n + 1) / 2; }

void platInit(Plat &p, Rng &rng, const FloatParams &fp) {
    if (p.type == PT_TRANSITION) { p.height = 5; return; }
    // EmptyPlatform::init
    p.length = randRange(4, 10, rng);
    if (p.width == -1) p.width = randRange(5, 9, rng);
    p.height = 5;
    switch (p.type) {
        case PT_WALL:
            p.wallHeight = randRange(P(fp, "obstaclesMinHeight"), P(fp, "obstaclesMaxHeight") + 1, rng);
            p.height = randRange(p.wallHeight + 4, p.wallHeight + 6, rng);
            break;
        case PT_LAVA: {
            p.length = randRange(6, 12, rng);
            const int minLava = std::min(P(fp, "obstaclesMinLava"), p.length - 2), maxLava = std::min(P(fp, "obstaclesMaxLava") + 1, p.length - 1);
            p.lavaLength = randRange(minLava, maxLava, rng);
            break;
        }
        case PT_STEP:
            p.stepHeight = randRange(P(fp, "obstaclesMinHeight"), P(fp, "obstaclesMaxHeight") + 1, rng);
            p.height = randRange(p.stepHeight + 2, p.stepHeight + 5, rng);
            break;
        case PT_GAP:
            p.gap = randRange(P(fp, "obstaclesMinGap"), std::min(P(fp, "obstaclesMaxGap") + 1, p.length - 1), rng);
            p.gapX = randRange(1, p.length - p.gap, rng);
            break;
        default: break;
    }
}

bool platMaxDifficulty(const Plat &p, const FloatParams &fp) {
    switch (p.type) {
        case PT_WALL: return p.wallHeight >= P(fp, "obstaclesMaxHeight");
        case PT_LAVA: return p.lavaLength >= P(fp, "obstaclesMaxLava");
        case PT_STEP: return p.stepHeight >= P(fp, "obstaclesMaxHeight");
        default: return false;
    }
}

int platRequiredBoxes(const Plat &p) {
    switch (p.type) {
        case PT_WALL: return tri(p.wallHeight - 1);
        case PT_LAVA: return std::max(1, p.lavaLength - 1);
        case PT_STEP: return tri(p.stepHeight - 1);
        case PT_GAP: return tri(std::max(0, p.gap - 2));
        default: return 0;
    }
}

void platGenerate(Plat &p, Rng &rng) {
    switch (p.type) {
        case PT_WALL: {
            p.addFloor(); p.addWalls();
            const int wallX = randRange(1, p.length, rng);
            const int wallThickness = randRange(1, p.length - wallX + 1, rng);
            p.layout.push_back({{wallX, 1, 1}, {wallX + wallThickness, 1 + p.wallHeight, p.width - 1}});
            for (int x = wallX; x < wallX + wallThickness; ++x)
                for (int z = 1; z < p.width; ++z) p.occupancy[{x, z}] = p.wallHeight;
            break;
        }
        case PT_LAVA: {
            p.addFloor(); p.addWalls();
            const int lavaX = randRange(1, p.length - p.lavaLength, rng);
            p.terrain.push_back({2, {{lavaX, 1, 1}, {lavaX + p.lavaLength, 2, p.width - 1}}});
            break;
        }
        case PT_STEP: {
            const int stepX = randRange(1, p.length, rng);
            p.layout.push_back({{0, 0, 0}, {stepX + 1, 1, p.width}});
            p.layout.push_back({{stepX, p.stepHeight, 0}, {p.length, p.stepHeight + 1, p.width}});
            p.layout.push_back({{stepX, 0, 0}, {stepX + 1, p.stepHeight + 1, p.width}});
            p.anchorLocal[0] = p.length; p.anchorLocal[1] = p.stepHeight; p.anchorLocal[2] = 0;
            p.addWalls();
            for (int x = stepX + 1; x < p.length; ++x)
                for (int z = 1; z < p.width; ++z) p.occupancy[{x, z}] = p.stepHeight;
            break;
        }
        case PT_GAP:
            p.layout.push_back({{0, 0, 0}, {p.gapX, 1, p.width}});
            p.layout.push_back({{p.gapX + p.gap, 0, 0}, {p.length, 1, p.width}});
            p.anchorLocal[0] = p.length; p.anchorLocal[1] = 0; p.anchorLocal[2] = 0;
            p.addWalls();
            break;
        case PT_EXIT:
            p.addFloor(); p.addWalls();
            p.terrain.push_back({1, {{p.length - 3, 1, 1}, {p.length - 1, 3, p.width - 1}}});
            break;
        default:
            p.addFloor(); p.addWalls();
            break;
    }
}

// Platform::generateObjectPositions / GapPlatform override (platforms.hpp:248-276,489-508)
std::vector<I3> platObjectPositions(Plat &p, int n, Rng &rng) {
    std::vector<I3> boxes;
    if (p.type == PT_GAP) {
        std::vector<I3> candidates;
        for (int x = 0; x < p.length; ++x)
            for (int z = 1; z < p.width - 1; ++z) {
                if (x >= p.gapX && x < p.gapX + p.gap) continue;
                candidates.push_back({x, 1, z});
            }
        for (int i = 0; i < n; ++i) {
            const I3 v = candidates[size_t(randRange(0, int(candidates.size()), rng))];
            const int y = ++p.occupancy[{v.x, v.z}];
            boxes.push_back({v.x, y, v.z});
        }
    } else {
        for (int i = 0; i < n; ++i)
            for (int attempt = 0; attempt < 10; ++attempt) {
                const int x = randRange(1, p.length - 1, rng);
                const int z = randRange(1, p.width - 1, rng);
                if (p.occupancy[{x, z}] < 2 || attempt >= 9) {
                    const int y = ++p.occupancy[{x, z}];
                    boxes.push_back({x, y, z});
                    break;
                }
            }
    }
    for (auto &c : boxes) c = p.root.applyCentre(c.x, c.y, c.z);  // adjustTransformation
    return boxes;
}

bool boxesCollide(const IBox &a, const IBox &b) {  // BoundingBox::collidesWith
    for (int k = 0; k < 3; ++k) {
        if (a.mx[k] <= b.mn[k]) return false;
        if (a.mn[k] >= b.mx[k]) return false;
    }
    return true;
}

}  // namespace

void LevelGenerator::generateObstacles(LevelOut &out) {
    MvLevel &L = out.level;
    Rng &rng = rng_;
    const int A = numAgents_;
    const FloatParams &fp = params_;
    std::vector<int> platformTypes = {PT_WALL, PT_LAVA, PT_STEP, PT_GAP};
    if (name_ == "obstacleswalls") platformTypes = {PT_WALL};
    else if (name_ == "obstaclessteps") platformTypes = {PT_STEP};
    else if (name_ == "obstacleslava") platformTypes = {PT_LAVA};

    const bool drawWalls = randRange(0, 2, rng);
    std::vector<Plat> platforms;
    int numPlatforms = 0;
    for (int attempt = 0; attempt < 20; ++attempt) {
        platforms.clear();
        numPlatforms = randRange(int(lroundf(fp.at("obstaclesMinNumPlatforms"))), int(lroundf(fp.at("obstaclesMaxNumPlatforms"))) + 1, rng);
        Plat start;
        start.type = PT_START; start.walls = W_SOUTH | W_EAST | W_WEST;
        platInit(start, rng, fp);
        platGenerate(start, rng);
        start.anchor = start.root.child(start.anchorLocal[0], start.anchorLocal[1], start.anchorLocal[2], 0);
        int requiredWidth = start.width;
        platforms.push_back(start);
        int prev = 0;
        int numMax = 0;
        const int allowedMax = int(fp.at("obstaclesNumAllowedMaxDifficulty"));
        for (int i = 0; i < numPlatforms; ++i) {
            const int orientation = randRange(0, 3, rng);  // STRAIGHT, TURN_LEFT, TURN_RIGHT
            requiredWidth = orientation == 0 ? requiredWidth : -1;
            Plat np;
            bool have = false;
            while (!have || (platMaxDifficulty(np, fp) && numMax >= allowedMax)) {
                np = Plat();
                np.type = platformTypes[size_t(randRange(0, int(platformTypes.size()), rng))];
                np.walls = W_WEST | W_EAST;
                np.width = requiredWidth;
                np.parent = platforms[size_t(prev)].anchor;
                np.root = np.parent;
                platInit(np, rng, fp);
                have = true;
            }
            if (platMaxDifficulty(np, fp)) ++numMax;
            platGenerate(np, rng);
            const int prevWidth = platforms[size_t(prev)].width;
            // rotateCCW: rotateYLocal(+90) then translateLocal(-1,0,-1); rotateCW: rotateYLocal(-90) then translateLocal(prevW-1, 0, -width+1)
            if (orientation == 1) np.root = np.parent.child(-1, 0, -1, 1);
            else if (orientation == 2) np.root = np.parent.child(prevWidth - 1, 0, -np.width + 1, 3);
            np.anchor = np.root.child(np.anchorLocal[0], np.anchorLocal[1], np.anchorLocal[2], 0);
            platforms.push_back(np);
            const int cur = int(platforms.size()) - 1;
            if (orientation != 0) {
                Plat tp;
                tp.type = PT_TRANSITION;
                tp.walls = W_NORTH | (orientation == 1 ? W_WEST : W_EAST);
                tp.length = platforms[size_t(cur)].width - 1; tp.width = prevWidth;
                tp.parent = platforms[size_t(prev)].anchor; tp.root = tp.parent;
                platInit(tp, rng, fp);
                platGenerate(tp, rng);
                tp.anchor = tp.root.child(tp.anchorLocal[0], tp.anchorLocal[1], tp.anchorLocal[2], 0);
                platforms.push_back(tp);
            }
            prev = cur;
            requiredWidth = platforms[size_t(cur)].width;
        }
        Plat ex;
        ex.type = PT_EXIT; ex.walls = W_NORTH | W_EAST | W_WEST; ex.width = requiredWidth;
        ex.parent = platforms[size_t(prev)].anchor; ex.root = ex.parent;
        platInit(ex, rng, fp);
        platGenerate(ex, rng);
        platforms.push_back(ex);

        bool selfCollision = false;
        for (int j = 0; j < int(platforms.size()) && !selfCollision; ++j)
            for (int k = 0; k < j - 2; ++k)
                if (boxesCollide(platforms[size_t(j)].outer(), platforms[size_t(k)].outer())) { selfCollision = true; break; }
        if (!selfCollision) break;
    }
    const uint32_t layoutColor = randomLayoutColor(rng);
    const uint32_t wallColor = randomLayoutColor(rng);

    VoxMap grid{100};
    const uint8_t wallType = uint8_t(MV_SOLID | (drawWalls ? MV_OPAQUE : 0));
    for (auto &p : platforms) {
        for (auto &b : p.layout) fillBox(grid, p.world(b), MV_SOLID | MV_OPAQUE, layoutColor);
        for (auto &b : p.wallBoxes) fillBox(grid, p.world(b), wallType, wallColor);
        std::vector<std::pair<int, IBox>> ts = p.terrain;
        std::stable_sort(ts.begin(), ts.end(), [](const std::pair<int, IBox> &a, const std::pair<int, IBox> &b) { return a.first < b.first; });
        for (auto &t : ts) fillTerrain(grid, p.world(t.second), t.first);
    }

    // StartPlatform::agentSpawnPoints (platforms.hpp:221-244)
    std::vector<I3> agentSpawn;
    {
        Plat &sp = platforms[0];
        std::set<std::pair<int, int>> used;
        for (int i = 0; i < A; ++i)
            for (int attempt = 0; attempt < 10; ++attempt) {
                const int x = randRange(1, sp.length - 1, rng);
                const int z = randRange(1, sp.width - 1, rng);
                if (used.count({x, z})) continue;
                const int y = sp.occupancy[{x, z}] + 1;
                sp.occupancy[{x, z}] += 2;
                agentSpawn.push_back({x, y, z});
                used.emplace(x, z);
                break;
            }
    }
    if (int(agentSpawn.size()) < A) throw std::runtime_error("start platform too small for the agents");

    std::vector<int> numBoxes(platforms.size(), 0);
    for (int i = 1; i < int(platforms.size()); ++i) {
        const int n = platRequiredBoxes(platforms[size_t(i)]);
        for (int box = 0; box < n; ++box) ++numBoxes[size_t(randRange(std::max(0, i - 2), i, rng))];
    }
    std::vector<I3> objs, rewards;
    for (int i = 0; i < int(platforms.size()); ++i) {
        const float randomBoxesFraction = frand(rng) * 0.5f;
        const int randomBoxes = int(lroundf(randomBoxesFraction * numBoxes[size_t(i)])) + randRange(0, 2, rng);
        const auto coords = platObjectPositions(platforms[size_t(i)], numBoxes[size_t(i)] + randomBoxes, rng);
        objs.insert(objs.end(), coords.begin(), coords.end());
    }
    for (int i = 1; i < int(platforms.size()) - 1; ++i) {
        const int numRewardObjects = randRange(0, 2, rng);
        const auto coords = platObjectPositions(platforms[size_t(i)], numRewardObjects, rng);
        rewards.insert(rewards.end(), coords.begin(), coords.end());
    }

    // DefaultScenario::spawnAgents
    for (int i = 0; i < A; ++i) {
        const float yaw = frand(rng) * 3.14159265358979323846f * 2;
        mvh::spawnBasis(yaw, L.spawn_basis[i]);
        const float sx = float(agentSpawn[size_t(i)].x) + 0.5f, sy = float(agentSpawn[size_t(i)].y) + 0.0f, sz = float(agentSpawn[size_t(i)].z) + 0.5f;
        L.spawn_pos[i][0] = sx; L.spawn_pos[i][1] = sy + 1.75f; L.spawn_pos[i][2] = sz;
        L.init_pos[i][0] = float(agentSpawn[size_t(i)].x); L.init_pos[i][1] = float(agentSpawn[size_t(i)].y); L.init_pos[i][2] = float(agentSpawn[size_t(i)].z);
    }

    // addEpisodeDrawables: merged boxes, terrain slabs (per platform, terrain-type order), objects, reward diamonds
    int ns = 0;
    for (const auto &g : mergeVoxels(grid)) {
        if (g.type == 0) continue;
        for (const auto &b : g.boxes) {
            MvBox &sb = staticAt(out, ns++);
            for (int a = 0; a < 3; ++a) {
                sb.h[a] = (float(b.mx[a] - b.mn[a] + 1) / 2) * 1.0f;
                sb.c[a] = (float(b.mn[a] + b.mx[a]) / 2 + 0.5f) * 1.0f;
            }
            sb.flags = g.type;
            sb.color = paletteIndex(g.color);
        }
    }
    L.n_static = ns;
    L.n_terrain = 0;
    for (auto &p : platforms) {
        std::vector<std::pair<int, IBox>> ts = p.terrain;
        std::stable_sort(ts.begin(), ts.end(), [](const std::pair<int, IBox> &a, const std::pair<int, IBox> &b) { return a.first < b.first; });
        for (auto &t : ts) {
            const IBox w = p.world(t.second);
            if (w.mx[0] - w.mn[0] > 0) {
                if (L.n_terrain >= MV_MAX_TERRAIN) throw std::runtime_error("too many terrain slabs");
                setTerrainModel(L.terrain[L.n_terrain], w, t.first == 1 ? C_LIGHT_GREEN : C_RED);
                L.terrain[L.n_terrain++].type = t.first;
            }
        }
    }
    if (int(objs.size()) > MV_MAX_OBJECTS - 1) throw std::runtime_error("too many movable objects");
    L.n_obj = int(objs.size());
    L.n_movable = int(objs.size());
    for (int i = 0; i < L.n_obj; ++i) {
        setStackingBox(L.obj_init[i], objs[size_t(i)]);
    }
    if (int(rewards.size()) > MV_MAX_REWARD) throw std::runtime_error("too many reward objects");
    L.n_reward = int(rewards.size());
    {
        using namespace mvh;
        // bottomHalf.rotateXLocal(180 deg).translate({0,-1,0})
        const float ang = 180.0f * 3.14159265358979323846f / 180.0f;
        M4 rx = identity();
        const float s = crsin(ang), c = crcos(ang);
        rx.c[1][1] = c; rx.c[1][2] = s; rx.c[2][1] = -s; rx.c[2][2] = c;
        const M4 bottom = mul(translation(0.0f, -1.0f, 0.0f), mul(identity(), rx));
        std::memcpy(L.cone_bottom_local, &bottom.c[0][0], 64);
        for (int i = 0; i < L.n_reward; ++i) {
            const I3 r = rewards[size_t(i)];
            L.reward_voxel[i][0] = int16_t(r.x); L.reward_voxel[i][1] = int16_t(r.y); L.reward_voxel[i][2] = int16_t(r.z);
            L.reward_voxel[i][3] = int16_t(paletteIndex(C_GREEN));
            const float tx = float(r.x) + 0.5f, ty = float(r.y) + 0.7f, tz = float(r.z) + 0.5f;
            const M4 root = mul(translation(tx, ty, tz), mul(scaling(0.17f * 0.8f, 0.45f * 0.8f, 0.17f * 0.8f), identity()));
            std::memcpy(L.reward_root[i], &root.c[0][0], 64);
        }
    }
    // ObstaclesScenario::episodeLengthSec (scenario_obstacles.cpp:262-266)
    L.episode_len = std::max(fp.at("episodeLengthSec"), float(numPlatforms) * 35 + float(objs.size()) * 1);
    L.n_movable = numPlatforms;  // reported by the level dump

    // dense grid bounds: every voxel entry, objects, rewards, one cell around; y from -30 (objects dropped into gaps sink
    // there).  Objects put down beyond the box are exact too (the step kernel's objAt finds them by their translation)
    int mn[3] = {1 << 20, -30, 1 << 20}, mx[3] = {-(1 << 20), -(1 << 20), -(1 << 20)};
    auto grow = [&](int x, int y, int z) { mn[0] = std::min(mn[0], x); mn[2] = std::min(mn[2], z); mx[0] = std::max(mx[0], x); mx[1] = std::max(mx[1], y); mx[2] = std::max(mx[2], z); };
    for (const auto &kv : grid) { const I3 c = voxUnkey(kv.first); grow(c.x, c.y, c.z); }
    for (auto &c : objs) grow(c.x, c.y, c.z);
    for (auto &c : rewards) grow(c.x, c.y, c.z);
    L.grid_org[0] = mn[0] - 1; L.grid_org[1] = mn[1]; L.grid_org[2] = mn[2] - 1;
    L.grid_dim[0] = mx[0] - mn[0] + 3; L.grid_dim[1] = mx[1] - mn[1] + 1 + 12; L.grid_dim[2] = mx[2] - mn[2] + 3;
    fillPlanes(out, &grid);
}

}  // namespace mv
