// Host-side procedural level generation (product code).
//
// Level layout depends on libstdc++'s mt19937 / uniform_int_distribution / uniform_real_distribution<float> /
// std::shuffle streams and on std::unordered_map iteration order, so it stays on the host, compiled with the same
// libstdc++ the reference uses (SURVEY.md Appendix C).  Each generator consumes the env's RNG in exactly the order
// Env::reset does (src/libs/env/src/env.cpp:57-76) and emits a flat MvLevel + bit-packed solid grid for the device.
#pragma once
#include <map>
#include <random>
#include <string>
#include <vector>

#include "mv_types.h"

namespace mv {

using FloatParams = std::map<std::string, float>;

// one entry of a level's draw sequence (insertion order of the reference's drawables); slots are assigned per mesh type
struct DrawRef { enum Kind { STATIC, TERRAIN, OBJECT, DECO, EYES, BARS, BODIES, REWARDS, REWARD_ONE } kind; int index; };  // REWARDS: all, as cone pairs

struct LevelOut {
    MvLevel level;
    std::vector<MvBox> statics;    // level.n_static layout boxes: collider order == draw order (std::map<BBoxInfo,Boxes> order); no bound
    std::vector<float> staticRot;  // two floats per static box (MV_ROTATED ones: local x axis in world space)
    std::vector<MvDeco> deco;      // level.n_deco static drawables with arbitrary model matrices
    std::vector<DrawRef> drawSeq;  // empty: the default order (opaque statics, terrain, objects, eyes, bars, bodies, rewards)
    std::vector<uint32_t> solid;  // grid_dim product bits, x-major: idx = (x*dimY + y)*dimZ + z
    std::vector<uint32_t> exitBits, lavaBits;  // terrain planes, same indexing
};

class LevelGenerator {
public:
    LevelGenerator(const std::string &scenarioName, int numAgents, const FloatParams &params);
    void seed(unsigned long s) { rng_.seed(s); }
    // the generator as constructed and then seeded: its stream starts again from its first level (Sokoban draws a fresh shuffle of its
    // level files instead of continuing the unplayed ones)
    void restart(unsigned long s) { rng_.seed(s); sokobanLevels_.clear(); }
    // Generates the next episode's level.  gridCells = capacity of the dense grid (cells); throws std::runtime_error
    // if the level does not fit one of the engine's fixed capacities (the number of static boxes is not one of them).
    void generate(LevelOut &out, int serial, int gridCells);
    // Same, but a level that does not fit a fixed capacity is replaced by the level the env's stream yields next instead of failing: up
    // to `attempts` draws.
    // Returns how many levels were skipped.  The env's level sequence then differs from the reference's from that episode on, which
    // is why the engine only does this when asked to (option "skip_unfit_levels").
    int generateFitting(LevelOut &out, int serial, int gridCells, int attempts = 8);

private:
    void generateTower(LevelOut &out);
    void generateObstacles(LevelOut &out);
    void generateCollect(LevelOut &out);
    void generateRearrange(LevelOut &out);
    void generateSokoban(LevelOut &out);
    void generateHexExplore(LevelOut &out);
    void generateHexMemory(LevelOut &out);
    void generateEmpty(LevelOut &out);
    unsigned episodeSeed_ = 0;     // the value the env reseeded itself with at this reset
    void assignSlots(LevelOut &out);
    void fillPlanes(LevelOut &out, const void *voxMap);
    int scenario_;
    std::string name_;
    int numAgents_;
    FloatParams params_;
    std::mt19937 rng_{std::random_device{}()};
    // Sokoban: Boxoban level files found at construction, and the shuffled levels not played yet (scenario_sokoban.cpp:39-116)
    std::vector<std::string> sokobanFiles_;
    std::vector<std::vector<std::string>> sokobanLevels_;
};

int scenarioFromName(const std::string &name);  // -1 if unknown
FloatParams defaultFloatParams(const std::string &scenarioName);
// default reward shaping of the (registered) scenario name
std::vector<std::pair<std::string, float>> defaultRewardShaping(const std::string &scenarioName);
// colour tables as the generators use them: [n all, n agent, n object, n layout], then the 0xRRGGBB values in that order (test pin)
std::vector<uint32_t> colorTables();
int gridCapacity(int scenario);
int decoCapacity(int scenario);  // most decorations a level of the scenario can hold  // dense voxel grid capacity in cells
int rewardSlot(int scenario, const std::string &key);  // -1 if unknown
const char *rewardKey(int scenario, int slot);         // the inverse for slots 1.. (nullptr: teamSpirit's slot 0, or no key of the scenario)

}  // namespace mv
