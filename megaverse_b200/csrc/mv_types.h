// Shared host/device plain-old-data layouts for the H100 voxel-world engine.
//
// HBM layout (one GPU, E envs, A agents per env, N = E*A views):
//   levels   MvLevel[E][2]          double-buffered immutable level description (host-generated, H2D on reset only); [bank rows] with "level_set"
//   statics  MvBox[E][2][staticCap] the levels' static layout boxes (collider order == draw order); staticCap grows on demand
//   staticRot float[E][2][staticCap][2]  MV_ROTATED boxes: local x axis in world space (ax, az)
//   solid    uint32[E][2][3][GW]    bit-packed voxel planes over the level's bounding grid: solid, exit terrain, lava terrain
//   objGrid  uint8[E][GC]           dynamic voxel -> movable-object id map (0xFF = none)
//   envs     MvEnvState[E]          per-env scalars + the building-zone set
//   agents   MvAgent[E*A]           kinematic controller + camera state
//   objects  MvObject[E][MAX_OBJ]   movable boxes
//   inst     MvInstance[E][MAX_INST] per-env drawable list in draw order (static part written at reset, dynamic part per step)
//   instCnt  int32[E][8]            {boxes, total, capsules, spheres, cones, cylinders, -, -}
//   views    float[N][16]           per-view camera matrices, written by the step kernel
//   obs      uint8[N][H][W][4]      the observation tensor (reference layout, megaverse.cpp:139-143)
//   depth    float[N][H][W]         optional
//   rewards float[N], dones uint8[E], trueObjectives float[N]
#pragma once
#include <stddef.h>
#include <stdint.h>

#define MV_MAX_AGENTS 8
#define MV_INITIAL_STATIC_CAP 768   // static boxes per level the engine starts with; it grows when a generated level needs more
#define MV_MAX_TERRAIN 16
#define MV_MAX_OBJECTS 128
#define MV_MAX_REWARD 128
#define MV_MAX_CAND 96      // per-agent collision candidates per step
#define MV_NO_OBJECT 0xFF

#define MV_SCENARIO_TOWER 0
#define MV_SCENARIO_OBSTACLES 1
#define MV_SCENARIO_COLLECT 2
#define MV_SCENARIO_REARRANGE 3
#define MV_SCENARIO_SOKOBAN 4
#define MV_SCENARIO_HEX_EXPLORE 5
#define MV_SCENARIO_HEX_MEMORY 6
#define MV_SCENARIO_EMPTY 7   // one static box, no rules: the scenario of the reference README's 75 k FPS figure (scenario_empty.cpp)

#define MV_MAX_DECO 1536    // static drawables that are not axis-aligned layout boxes (other meshes, rotated boxes); stored beside MvLevel
#define MV_MAX_ARRANGEMENT 8

// voxel / box flags (voxel_state.hpp:10-15)
#define MV_SOLID 1
#define MV_OPAQUE 2
#define MV_ROTATED 4   // static collider rotated about Y: MvLevel::static_rot holds its local x axis (ax, az)

// action bits (env.hpp:22-42)
#define MV_A_LEFT (1 << 1)
#define MV_A_RIGHT (1 << 2)
#define MV_A_FORWARD (1 << 3)
#define MV_A_BACKWARD (1 << 4)
#define MV_A_LOOKLEFT (1 << 5)
#define MV_A_LOOKRIGHT (1 << 6)
#define MV_A_JUMP (1 << 7)
#define MV_A_INTERACT (1 << 8)
#define MV_A_LOOKDOWN (1 << 9)
#define MV_A_LOOKUP (1 << 10)

// reward table slots (scenario_tower_building.hpp:44-52)
#define MV_R_TEAM_SPIRIT 0
#define MV_R_TOWER_PICKED_UP 1
#define MV_R_TOWER_VISITED_BZ 2
#define MV_R_TOWER_BUILDING 3
// Obstacles (scenario_obstacles.hpp:37-45)
#define MV_R_OBST_AGENT_AT_EXIT 1
#define MV_R_OBST_ALL_AT_EXIT 2
#define MV_R_OBST_EXTRA 3
#define MV_R_OBST_CARRIED_TO_EXIT 4
// Collect (scenario_collect.hpp:42-50)
#define MV_R_COLLECT_GOOD 1
#define MV_R_COLLECT_BAD 2
#define MV_R_COLLECT_ALL 3
#define MV_R_COLLECT_ABYSS 4
#define MV_R_REARRANGE_ONE_MORE 1
#define MV_R_REARRANGE_ALL 2
#define MV_R_SOKOBAN_ON_TARGET 1
#define MV_R_SOKOBAN_LEAVES_TARGET 2
#define MV_R_SOKOBAN_ALL 3
#define MV_R_EXPLORE_SOLVED 1
#define MV_R_MEMORY_GOOD 1
#define MV_R_MEMORY_BAD 2
#define MV_R_COUNT 8

// fault bits (per env, sticky): the engine never exit()s, it reports
#define MV_FAULT_LEVEL_NOT_READY 1   // episode ended before the host delivered the next level
#define MV_FAULT_TRI_OVERFLOW 2      // a view produced more triangles than the rasteriser's shared-memory list holds
#define MV_FAULT_GRID_RANGE 4        // a Sokoban box was pushed outside the dense voxel grid (walled rooms: not expected); objects put
                                     // down outside the grid are exact (the step kernel finds them by their translation)
#define MV_FAULT_NAN 8               // NaN position (agent.cpp:82-93 guard)
#define MV_FAULT_CAND_OVERFLOW 32     // more than MV_MAX_CAND colliders near one agent
#define MV_FAULT_ENVELOPE 16         // an agent left the per-step collision envelope the candidate colliders were culled against

struct MvBox {       // static layout box: drawable (OPAQUE) and/or collider (SOLID)
    float c[3];      // centre  = ((min+max)/2 + 0.5) * voxelSize        (layout_utils.cpp:30-34)
    float h[3];      // half extents = (max-min+1)/2 * voxelSize          (layout_utils.cpp:24-28)
    int32_t flags;   // MV_SOLID | MV_OPAQUE | (instance slot among the opaque boxes << 8)
    int32_t color;   // palette index
};

struct MvObjInit {   // a movable object at episode start
    int16_t voxel[3];
    int16_t color;   // palette index
    float scale[3];  // local scale (0.39 for the stacking boxes, component_object_stacking.hpp:172)
    int32_t meta;    // MvObject::meta
    float pos[3];    // local translation (voxel + 0.5 for objects that sit in the middle of their voxel)
};

struct MvDeco {      // static drawable with an arbitrary model matrix
    float model[16];
    int32_t mesh, color, slot, pad;
};

struct MvTerrain {
    float model[16];  // column-major model matrix (layout_utils.cpp:53-68)
    int32_t color;
    int32_t type;     // TerrainType bit (platforms.hpp:28-34)
    int32_t bb[6];    // world voxel box min3, max3 (exclusive)
};

struct MvLevel {
    int32_t serial;       // episode index this level belongs to (checked by the device reset)
    int32_t scenario;
    int32_t n_static, n_terrain, n_obj;
    int32_t n_movable;    // numMovableBoxes() for episodeLengthSec (scenario_tower_building.cpp:263-266)
    int32_t grid_org[3], grid_dim[3];
    int32_t bz_min[3], bz_max[3];  // building zone (x,z used)
    float episode_len;             // episodeLengthSec() of this level (scenario_tower_building.cpp:263-266, scenario_obstacles.cpp:262-266)
    float look_limit;              // floatParams["verticalLookLimitRad"]
    int32_t n_reward;              // Obstacles / Collect: reward diamonds
    int32_t n_positive;            // Collect: numPositiveRewards
    int32_t n_opaque;              // number of drawable static boxes (their instance slot is flags >> 8)
    int32_t n_static_pre;          // statics[0 .. n_static_pre) precede the movable objects in collider order, the rest follow them
    // instance-list layout, assigned by the host so that the list is in the reference's draw order (mesh type major,
    // insertion order minor): first slot of the terrain slabs, agents' eyes / HUD bars / bodies, reward cones; totals per mesh
    int32_t slot_terrain, slot_eyes, slot_bars, slot_body, slot_reward;
    int32_t mesh_counts[5];        // box, capsule, sphere, cone, cylinder instances
    int32_t n_deco;
    int32_t n_arr;                 // Rearrange: target arrangement items
    int16_t arr[MV_MAX_ARRANGEMENT][6];  // mesh, palette colour, offset x y z from the centre
    int32_t work_center[3];        // Rearrange: rightCenter
    float goal[3];                 // HexExplore: rewardObjectCoords
    int32_t n_grid_static;         // statics[0 .. n_grid_static) are the merged boxes of the voxel grid (the rest are free-standing boxes)
    int32_t pad0[1];
    // the static boxes themselves live beside the level (StepParams::statics / staticRot): their number has no bound in the reference
    // (component_voxel_grid.hpp:108-187), so the engine sizes that array at run time
    MvTerrain terrain[MV_MAX_TERRAIN];
    MvObjInit obj_init[MV_MAX_OBJECTS];
    float spawn_pos[MV_MAX_AGENTS][4];     // ghost origin at spawn (agent.cpp:45)
    float spawn_basis[MV_MAX_AGENTS][12];  // ghost basis rows (btMatrix3x3(btQuaternion(Y, yaw)))
    float init_pos[MV_MAX_AGENTS][4];      // FallDetection agentInitialPositions
    int16_t reward_voxel[MV_MAX_REWARD][4];  // reward objects: voxel + palette colour (Collect: GREEN = +1, RED = -1)
    float reward_root[MV_MAX_REWARD][16];    // addDiamond root model matrix (layout_utils.cpp:114-126)
    float cone_bottom_local[16];             // the lower cone's local transform (rotateXLocal(180 deg), translate(0,-1,0))
    // per reward object: first instance slot, mesh, number of instances (1 sphere, 2 cones, 3 cylinders = pillar with two caps),
    // goodness (HexMemory); pillars keep their caps' local transforms (setParentKeepTransformation, layout_utils.cpp:100-112)
    int16_t reward_slot[MV_MAX_REWARD];
    int8_t reward_mesh[MV_MAX_REWARD], reward_cnt[MV_MAX_REWARD];
    uint32_t reward_good[4];
    float reward_child[MV_MAX_REWARD][2][16];
};

struct MvAgent {
    float pos[3];
    float basis[9];  // rows
    float hvel[3];
    float vvel, voff, step_off, jump_speed;
    float jump_axis[3];
    float cur_x;
    float cam_local[16];
    float bar_scale[3];
    float total_reward;
    float object_t[16];  // agent Object3D transformation (updateTransform)
    int32_t was_on_ground, was_jumping, carrying, picked_up, visited_bz;
    int32_t pad[2];
};

struct MvObject {
    float t[3];      // local translation
    float s[3];      // local scale (matrix diagonal)
    float col_c[3];  // collider centre / half extents (RigidBody::syncPose, physics.hpp:69-74)
    float col_h[3];
    int32_t parent;  // -1 scene, else agent index (child of its pickupSpot)
    int32_t enabled; // collider responds (CF_NO_CONTACT_RESPONSE cleared)
    int32_t color;
    int32_t meta;    // bits 0..2 mesh, bits 3..5 collision class (0: scale 1.15 offset (0,-0.05,0); 1: scale 1; 2: scale (1,0.5,1);
                     // 3: scale (1,2,1); 4: scale (1.15,3,1.15) offset (0,0.6,0)), bits 8.. instance slot
};
#define MV_OBJ_MESH(meta) ((meta) & 7)
#define MV_OBJ_COLCLASS(meta) (((meta) >> 3) & 7)
#define MV_OBJ_SLOT(meta) ((meta) >> 8)

struct MvEnvState {
    float episode_sec;
    int32_t num_frames;
    int32_t episode_idx;
    int32_t slot;            // the live slot of the env's ring of level slots; with option "level_set" the env's live row of the bank
    int32_t highest_tower;
    float bz_reward;         // currBuildingZoneReward
    int32_t faults;
    // std::unordered_set<VoxelCoords> objectsInBuildingZone, emulated in libstdc++ iteration order (bzset.h)
    int32_t solved;          // Obstacles: all agents reached the exit
    uint32_t reached_exit;   // Obstacles: bit per agent; Rearrange: maxMatchingObjects
    uint32_t reward_alive[4];  // bit per reward object still in place
    int32_t positive_collected;  // Collect; Sokoban: numBoxesOnGoal
    int32_t bz_count, bz_nb, bz_next_resize;
    int16_t bz_items[MV_MAX_OBJECTS][4];
    int32_t pad[2];          // pad[0]: with option "level_set" the env's pick seed (uint32 bits), set by the host, never by the kernel; pad[1]: with
                             // option "autoreset" 1 or 2, 1 from the call in which the episode ended to the flip that starts the next (else 0)
};

// One drawable of an env, in the reference's draw order (mesh type major, insertion order minor,
// v4r_env_renderer.cpp:267-279): boxes first (static layout, terrain slabs, movable objects, agents' eyes, HUD bars),
// then capsules (agent bodies), spheres, cones, cylinders.  Static entries are written at episode reset, dynamic ones
// every step by the step kernel; the rasteriser is scenario-agnostic and only reads this list + the view matrices.
struct MvInstance {
    float model[16];  // column-major absoluteTransformationMatrix()
    int32_t mesh;     // 0 box, 1 capsule, 2 sphere, 3 cone, 4 cylinder (DrawableType, env.hpp:57-67)
    int32_t color;    // palette index
    int32_t pad[2];   // pad[0]: segmentation tag MV_SEG_* << 8 | index (written by the step kernel, read by the rasteriser); pad[1]: 0
};
// instance slots besides the static boxes and decorations: the engine allocates staticCap + MV_DYN_INSTANCES + the scenario's decoration
// capacity per env; the rasteriser's draw-order key bounds the total at MV_HARD_MAX_INSTANCES
#define MV_DYN_INSTANCES (MV_MAX_TERRAIN + MV_MAX_OBJECTS + 3 * MV_MAX_AGENTS + 3 * MV_MAX_REWARD)
#define MV_HARD_MAX_INSTANCES 32767

struct MvConsts {        // host-computed constants (so host libm decides their bits once, identically for oracle and device)
    float look_left[9];  // btMatrix3x3(btQuaternion(Y, +3.5*dt)) rows
    float look_right[9];
    float max_slope_cos; // btCos(btRadians(45))
    float p00, p11, p22, p32;  // V4R projection (v4r.cpp:35-45)
    float dt;
    float reward_default[MV_R_COUNT];
};

#ifdef __cplusplus
static_assert(sizeof(MvBox) == 32 && sizeof(MvObject) == 64, "TMA bulk copies need 16-byte multiples");
static_assert(sizeof(MvLevel) % 16 == 0, "MvLevel alignment");
static_assert(sizeof(MvInstance) == 80, "MvInstance layout");
static_assert(sizeof(MvEnvState) % 4 == 0 && sizeof(MvAgent) % 4 == 0, "word copies");
#endif
