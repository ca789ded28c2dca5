/* megaverse_b200 -- thin C ABI of the H100 batched voxel-world step + render engine.
 *
 * Drop-in boundary for the reference's per-step hot path.  Each entry point replaces what the reference's pybind11
 * class MegaverseGym (src/libs/bindings/megaverse.cpp:36-263) reaches through VectorEnv (src/libs/env/src/vector_env.cpp)
 * and EnvRenderer (src/libs/env/include/env/env_renderer.hpp:12-32).  Plain pointers and sizes only; no torch / pybind
 * types.  Every call returns 0 on success or a negative MV_ERR_* code; mv_last_error() gives the message.  The engine
 * never calls exit() (the reference's TLOG(FATAL) does, src/libs/util/src/tiny_logger.cpp:109-113).
 *
 * Threading: calls on one handle must be serialised by the caller (the reference holds the GIL for every call).
 * Observation memory is owned by the engine and reused every step, exactly like the reference's renderer buffer
 * (megaverse.cpp:139-143): pointers stay valid until mv_close, contents until the next mv_step / mv_reset.
 */
#ifndef MEGAVERSE_B200_H
#define MEGAVERSE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mv_engine *mv_handle;

#define MV_OK 0
#define MV_ERR_ARG -1          /* bad argument (unknown scenario, bad sizes, unknown reward key -> std::out_of_range in the reference) */
#define MV_ERR_CUDA -2         /* CUDA runtime failure, or no CUDA device: the product has NO CPU fallback */
#define MV_ERR_CAPACITY -3     /* a generated level exceeds the engine's fixed capacities */
#define MV_ERR_STATE -4        /* call order (e.g. step before reset) */

/* why an episode ended (mv_done_reasons): one byte per env and step, beside the done flag */
#define MV_END_NONE 0          /* not done (also every env after mv_reset, and the envs mv_reset_envs restarted) */
#define MV_END_TIME 1          /* the episode clock ran out: truncated */
#define MV_END_SOLVED 2        /* a scenario rule solved the level (doneWithTimer), also when a request or the clock ends it in the
                                * 0.3 s grace that follows: terminal */
#define MV_END_REQUESTED 3     /* the caller's end mask (mv_step_device_ends): truncated */

/* segmentation classes (option "segmentation"): a pixel's value is class << 8 | index, 0 where nothing was drawn */
#define MV_SEG_NONE 0          /* background: nothing drawn (depth 0) */
#define MV_SEG_STATIC 1        /* static layout boxes and static decorations (hex-maze walls, Rearrange's target arrangement, ...); index 0 */
#define MV_SEG_TERRAIN 2       /* terrain slabs; index = the slab's TerrainType bit number (0 exit, 1 lava, 2 building zone) */
#define MV_SEG_OBJECT 3        /* movable objects, carried or not; index = the object's index in the level's object list */
#define MV_SEG_AGENT 4         /* an agent's body, eyes and HUD bar; index = agent index within the env */
#define MV_SEG_REWARD 5        /* reward objects (diamonds, Collect's objects, hex-maze objects, pillars); index = reward-object index */

/* MegaverseGym::MegaverseGym (megaverse.cpp:38-58).  num_threads = host level-generation workers (the reference's
 * numSimulationThreads drove Bullet on the CPU, vector_env.cpp:6-40).  device = CUDA ordinal. */
int mv_create(const char *scenario, int w, int h, int num_envs, int num_agents_per_env, int num_threads, int device,
              const char *const *param_keys, const float *param_vals, int nparams, mv_handle *out);
/* Mixed-scenario engine (a multi-task batch, e.g. Megaverse-8, in ONE engine: one step kernel and one raster launch per step for all
 * envs).  scenarios[e] names env e's scenario: any registered name (case-insensitive), repeated in any layout.  One render size, agent
 * count and params dict for every env: each env starts from its own scenario's defaults and then takes the overrides.  Env e behaves
 * exactly as env e of a single-scenario engine of its name (same levels, frames, rewards, dones for the same seed and actions), and
 * reward shaping (mv_get / mv_set_reward_shaping) uses the keys of the env's scenario.  mv_create is this call with num_envs copies
 * of one name.  Errors (MV_ERR_ARG, before any CUDA call): a null list, a null or unknown name (the message names the env), bad sizes,
 * useUIRewardIndicators > 0.
 * Memory: the per-env arrays keep one pitch per engine, that of the largest capacity among its scenarios.  With any Obstacles env in
 * the batch every env costs 512 KiB of object grid plus 384 KiB of bit planes in HBM and 384 KiB of pinned host staging (1 024 envs:
 * about 0.9 GiB of HBM and 384 MiB pinned); state-store rows grow to match (mv_state_row_bytes). */
int mv_create_mixed(const char *const *scenarios, int w, int h, int num_envs, int num_agents_per_env, int num_threads, int device,
                    const char *const *param_keys, const float *param_vals, int nparams, mv_handle *out);
/* message of the last failed call; pass NULL for a failed mv_create */
const char *mv_last_error(mv_handle h);

/* MegaverseGym::seed (megaverse.cpp:60-69): master mt19937 -> one randRange(0,1<<30) per env */
int mv_seed(mv_handle h, int seed);
/* Env::seed for one env (megaverse_test_app.cpp:250-254 seeds env i with 42+i) */
int mv_seed_env(mv_handle h, int env, int seed);

/* MegaverseGym::reset -> VectorEnv::reset (vector_env.cpp:110-120): new episode in every env + first render */
int mv_reset(mv_handle h);

/* MegaverseGym::setActions for all agents at once: masks[env*A + agent] = Action bit mask (env.hpp:22-42).
 * mv_encode_action converts one 6-tuple of Discrete heads {3,3,3,2,2,3} exactly like megaverse.cpp:100-116. */
int mv_set_actions(mv_handle h, const int32_t *masks);
int32_t mv_encode_action(const int32_t *heads6);

/* MegaverseGym::step -> VectorEnv::step (vector_env.cpp:89-108): physics + scenario logic, reset of finished envs, render.
 * Synchronous: on return observations / rewards / dones are in host memory. */
int mv_step(mv_handle h);
/* mv_step in two halves, for a double-buffered consumer (two engines of half the envs each, the arrangement Sample Factory's
 * sampler uses with two env groups per worker: while the policy looks at group A, group B steps).  mv_step_begin uploads the
 * action masks and enqueues the kernels and the device->host copies, then returns; mv_step_end waits for them and does the
 * episode bookkeeping -- on return the host buffers are valid exactly as after mv_step.  With option "zero_copy" 0 the
 * observation tensor travels by the copy engine, which overlaps with the other engine's kernels.  Any other call that needs a
 * finished step (mv_reset, mv_step_device, mv_fetch_obs) ends an outstanding begin first; a second begin is MV_ERR_STATE. */
int mv_step_begin(mv_handle h);
int mv_step_end(mv_handle h);
/* Steps with an active set: only the chosen envs advance.  In such a call an INACTIVE env does nothing: it runs no tick (at any
 * action_repeat), its env, agent, object and grid state, episode clock and step counter, level slots, instance lists and camera views are
 * unchanged, its action masks and its end request (d_ends) are ignored, and no level is generated or uploaded for it.  It reports reward 0
 * for each of its agents, done 0 and reason MV_END_NONE, its true objectives unchanged, and no terminal frame.  Its views' rows in every
 * engine-owned output buffer the call delivers to still hold its current frame: obs, and depth and segmentation when they are on -- the pinned
 * host buffers for mv_step_envs, HBM for mv_step_device_active, and the copy mv_fetch_obs makes.  An ACTIVE env is stepped exactly as by the
 * corresponding full call (action repeat, end requests, level slots, terminal frames, depth, segmentation, mixed engines): env e delivers
 * over any sequence of such calls what env e of an engine with the same seeds and options delivers when it is stepped by mv_step (or
 * mv_step_device_ends with the same requests) only at the calls where e was active.  The asynchronous call's contract (three calls per
 * episode with two level slots) counts calls as before: an inactive env cannot end.
 * The raster launch draws only the active envs' views when its destination already holds every view's current frame: the pinned host
 * buffers after host-facing calls and the re-renders of mv_reset / mv_reset_envs / mv_states_load, but not after mv_step_device* until
 * mv_fetch_obs; the engine's own HBM buffers after a call that drew into them.  A caller-owned buffer (mv_set_obs_buffer) always has every
 * view drawn: the engine cannot vouch for its rows.  Otherwise every view is drawn; only the step is masked.  mv_last_kernel_ms and
 * mv_kernel_launches read as for the corresponding full call.  mv_step_begin / mv_step_end always step every env.
 * mv_step_envs: the synchronous, host-facing call, like mv_step, with an EnvPool-style list envs[0..n): the listed envs are active.  Actions
 * come from mv_set_actions; the entries of unlisted envs are ignored.  n == 0 is a call in which every env is inactive.  MV_ERR_ARG (n < 0, a
 * null list with n > 0, an env out of range or listed twice) and MV_ERR_STATE (before mv_reset, an outstanding mv_step_begin) change
 * nothing. */
int mv_step_envs(mv_handle h, const int32_t *envs, int n);

/* MegaverseGym::getObservation (megaverse.cpp:139-143): uint8[N][h][w][4] RGBA, view index env*A+agent, host memory */
int mv_obs_host(mv_handle h, const uint8_t **out);
/* float32[N][h][w] view-space depth (V4R depth output definition), only when option "depth" is 1 */
int mv_depth_host(mv_handle h, const float **out);
/* MegaverseGym::getLastRewards (megaverse.cpp:128-137): float[N] */
int mv_rewards(mv_handle h, const float **out);
/* VectorEnv::done (vector_env.hpp): uint8[num_envs] */
int mv_dones(mv_handle h, const uint8_t **out);
/* VectorEnv::trueObjectives / MegaverseGym::trueObjective (megaverse.cpp:209-212): float[N] */
int mv_true_objectives(mv_handle h, const float **out);
/* uint8[num_envs] MV_END_* of the last step, host memory, valid like mv_dones (non-zero exactly where dones is 1).  A state-store row carries
 * them: after mv_states_load they read as after the saved step. */
int mv_done_reasons(mv_handle h, const uint8_t **out);
/* Terminal frames, option "final_obs" (before the first reset).  For every env that ends in a step (dones[e] == 1), views e*A .. e*A+A-1
 * of the final-frame buffer get the frame that step would have drawn had the episode not ended: the scene after this step's actions,
 * physics, scenario rules and HUD update, before the flip to the next level -- the s_T a truncated episode is bootstrapped from.  Same
 * size and layout as the observation tensor (and the depth tensor when option depth is on).  Rows of envs that did not end are not
 * written: a row keeps the terminal frame of the env's last end.
 * Host-facing steps (mv_step, mv_step_begin/end with obs_to_host 1) store the rows straight into the host buffer (mv_final_obs_host), on
 * return like the observations; mv_step_device[_ends] stores them into the device buffer (mv_final_obs_device) in stream order, and
 * mv_fetch_obs then copies the whole device buffer into the host one.  mv_reset, mv_reset_envs and mv_states_load draw no terminal frame.
 * Nothing else changes with the option: obs, depth, rewards, dones and true objectives are byte-identical with it on and off.
 * Cost: a device and a pinned host buffer each as large as the observation tensor (+ depth), e.g. 151 MB each at Collect 1 024 x 4 and
 * 128 x 72, and one more instance row per env in HBM: 552 + static_cap + decoration slots of 80 B, 103 KiB per env at the default
 * static_cap (223 KiB in the hex mazes, whose decorations take 1 536 slots).  Time: one raster launch per step that draws only the ended
 * envs' views, and the ending envs' warps write their terminal rows (DESIGN.md section 3 has the measured costs).
 * MV_ERR_ARG when the option (or, for depth, option depth) is off; MV_ERR_STATE before mv_reset. */
int mv_final_obs_host(mv_handle h, const uint8_t **out);
int mv_final_depth_host(mv_handle h, const float **out);
int mv_final_obs_device(mv_handle h, uint8_t **d_final_obs);
int mv_final_depth_device(mv_handle h, float **d_final_depth);
/* Segmentation, option "segmentation" (0/1, before the first reset: MV_ERR_STATE after it, MV_ERR_ARG for any other value; default 0).
 * uint16[N][h][w], view index env*A + agent, rows as in the observation tensor: the MV_SEG_* class of the drawable behind each pixel << 8 |
 * its index, 0 exactly where nothing was drawn (exactly where depth is 0).  The rasteriser names the drawable whose fragment won the pixel,
 * so the tensor shows coverage and the depth-tie order exactly, in both shading modes.  Every call that draws the batch writes it beside
 * the observations and is delivered the same way: mv_step and mv_step_begin/end into the host buffer (mv_segmentation_host), on return
 * like the observations; mv_step_device[_ends] into the device buffer (mv_segmentation_device) in stream order, copied down by
 * mv_fetch_obs; mv_reset, mv_reset_envs and mv_states_load draw it again.  Nothing else changes with the option: obs, depth, rewards,
 * dones, done reasons, true objectives and terminal frames are byte-identical with it on and off.
 * Memory: 2 B per pixel in HBM and again pinned (18 432 B per view at 128 x 72: 75.5 MB each at Collect 1 024 x 4); nothing is
 * allocated while the option is off.
 * Limits: mv_draw_hires and mv_debug_render_instances draw no segmentation (the debug call mv_debug_render_instances_ex can, with its
 * own tags); mv_set_obs_buffer does not redirect it (it stays in the
 * engine's own buffer); terminal frames (option final_obs) carry none; the multi-GPU gather does not gather it.
 * Both calls return MV_ERR_ARG when the option is off; the device pointer is refused (MV_ERR_STATE) exactly when mv_depth_device's is. */
int mv_segmentation_host(mv_handle h, const uint16_t **out);
int mv_segmentation_device(mv_handle h, uint16_t **d_seg);
/* State tensors, option "state_tensors" (0/1, before the first reset: MV_ERR_STATE after it, MV_ERR_ARG for any other value; default 0).
 * The state behind the frames, written by the step kernel in the same call: four float32 tensors whose every value is a bit copy of an
 * engine field (integers are stored exactly, all are below 2^24).
 *   agents  [N][16], row env*A + agent: 0-2 MvAgent::pos; 3-6 the yaw block of the ghost basis, basis[0], basis[2], basis[6], basis[8] (the
 *           controller's forward is normalise(b6, b7, -b8)); 7 cur_x (camera pitch, radians); 8-10 hvel; 11 vvel; 12 was_on_ground;
 *           13 was_jumping; 14 carrying (object index, -1 = none); 15 total_reward
 *   envs    [E][16]: 0 episode_sec; 1 episode_len of the live level; 2 num_frames; 3 scenario (MV_SCENARIO_*); 4 n_obj; 5 n_reward; 6 solved;
 *           7 reached_exit; 8 highest_tower; 9 bz_reward; 10 positive_collected; 11-15 0
 *   objects [E][128][4] (MV_MAX_OBJECTS): rows < n_obj: world position x, y, z -- the translation column of the model matrix the object is
 *           drawn with, ((agent * camera) * pickup) * local for a carried one, as mv_debug_get_state reports it -- then the carrier
 *           (MvObject::parent: agent index, -1 when not carried); rows beyond are 0
 *   rewards [E][128][4] (MV_MAX_REWARD): rows < n_reward: the translation of the reward object's root matrix, then 0 once it is collected,
 *           else -1 for a penalising object (Collect: not GREEN; HexMemory: a bad object) and +1 otherwise; rows beyond are 0
 * A row shows the state the returned frame shows: for an env that ended in the call, the new episode's first.  Inactive envs (mv_step_envs,
 * mv_step_device_active) keep their rows; mv_reset and mv_reset_envs write the restarted envs' rows; mv_states_load restores the saved
 * step's rows (the state store carries them: mv_state_row_bytes grows by 64 * A + 4 160 bytes with the option on); mv_debug_warp_agent
 * changes no row until the next call.  With option final_obs as well, an env that ends in a step gets terminal rows in four more tensors of
 * the same shapes: the state after the ending tick, before the flip -- the state its terminal frame shows.  Other rows are left alone.
 * Delivery follows the observations: host-facing calls (mv_step, mv_step_envs, mv_step_begin/end, mv_reset, mv_reset_envs, mv_states_load)
 * return with every tensor in pinned host memory (one copy of the whole block, on a copy stream while the frames are drawn);
 * mv_step_device* leaves them in HBM in stream order, and mv_fetch_obs copies them down.  Nothing else changes with the option: obs,
 * depth, segmentation, rewards, dones, reasons, true objectives, terminal frames and level ids are byte-identical with it on and off.
 * Memory: 64 * A + 4 160 B per env in HBM and again pinned (4.5 MB each at 1 024 envs x 4 agents), twice that with final_obs; nothing is
 * allocated while the option is off.  Any out pointer may be NULL.  MV_ERR_ARG for a null handle and while the option (or, for the
 * terminal rows, option final_obs) is off; MV_ERR_STATE before mv_reset. */
#define MV_STATE_OBJECT_ROWS 128
#define MV_STATE_REWARD_ROWS 128
int mv_state_tensors_host(mv_handle h, const float **agents, const float **envs, const float **objects, const float **rewards);
int mv_state_tensors_device(mv_handle h, float **agents, float **envs, float **objects, float **rewards);
int mv_final_state_tensors_host(mv_handle h, const float **agents, const float **envs, const float **objects, const float **rewards);
int mv_final_state_tensors_device(mv_handle h, float **agents, float **envs, float **objects, float **rewards);
/* Ray sensors: every agent casts the same fan of n rays against its env's drawn scene, and each ray reports the distance to the first
 * surface it meets and what that surface is.
 * mv_set_rays, before the first reset (MV_ERR_STATE after it): dirs3 = float[n][3], directions in CAMERA space, the frame of the agent's
 * view matrix (x right, y up, -z forward); n = 0 turns the rays off (the default), else 1..MV_MAX_RAYS; max_dist finite and > 0.  A
 * direction that is zero or not finite, n out of range or a bad max_dist is MV_ERR_ARG and changes nothing.  Each direction is used
 * exactly as given, and a distance counts multiples of its length: unit vectors give world units.  One fan for every agent of the engine,
 * in single-scenario and mixed engines alike (megaverse_b200/rays.py builds fans and rings).
 * What a ray hits: every entry of the env's instance list that the rasteriser draws (the same rows and counts), meshes as drawn (boxes are
 * the cube [-1, 1]^3), front faces only -- a ray that starts inside a box or a closed mesh does not hit it -- except the agent's own body,
 * eyes and HUD bar (tag MV_SEG_AGENT << 8 | own index).  The hit is the nearest; on an exact tie the later entry in draw order wins, as
 * the rasteriser's LESS_OR_EQUAL does.  The arithmetic is defined operation by operation in DESIGN.md section 3 ("Ray sensors"), so that
 * a CPU restatement gives the same bits.
 * Outputs, ray r of view env*A + agent at [view][r]: dist float[N][n], the hit's parameter t along the direction (0: no hit within
 * max_dist); tag uint16[N][n], the hit drawable's MV_SEG_* class << 8 | index (0: no hit) -- the conventions of depth and segmentation.
 * Rays always describe the scene the current frames show: every call that draws the step's frames writes them (mv_step,
 * mv_step_begin/end, mv_step_envs, mv_step_device[_ends|_active], mv_reset, mv_reset_envs, mv_states_load's redraw), after the last tick
 * with action_repeat; inactive envs keep theirs.  With option final_obs as well, an env that ends in a step gets terminal rays, cast from
 * the terminal rows its terminal frame is drawn from; other terminal rows are left alone.
 * Delivery: host-facing calls return with both arrays in pinned host memory (mv_rays_host; one copy on the step's stream);
 * mv_step_device* leaves them in HBM (mv_rays_device) in stream order, and mv_fetch_obs copies them down.  Nothing else changes: obs,
 * depth, segmentation, rewards, dones, reasons, true objectives, terminal frames and state tensors are byte-identical with rays on and off.
 * Cost: one launch per drawing call (two with terminal rays); 6 B per ray per view in HBM and again pinned, twice that with final_obs.
 * The getters take NULL out pointers; MV_ERR_ARG for a null handle and while the rays (or, for the terminal rays, option final_obs) are
 * off; MV_ERR_STATE before mv_reset. */
#define MV_MAX_RAYS 256
int mv_set_rays(mv_handle h, const float *dirs3, int n, float max_dist);
int mv_rays_host(mv_handle h, const float **dist, const uint16_t **tag);
int mv_rays_device(mv_handle h, float **dist, uint16_t **tag);
int mv_final_rays_host(mv_handle h, const float **dist, const uint16_t **tag);
int mv_final_rays_device(mv_handle h, float **dist, uint16_t **tag);

/* MegaverseGym::getRewardShaping / setRewardShaping (megaverse.cpp:214-222).  get: fills up to cap entries, returns the
 * number of keys in *n.  Key strings are owned by the engine. */
int mv_get_reward_shaping(mv_handle h, int env, int agent, const char **keys, float *vals, int cap, int *n);
int mv_set_reward_shaping(mv_handle h, int env, int agent, const char *const *keys, const float *vals, int n);

/* options: "depth" (0/1, before first reset), "obs_to_host" (0/1: whether mv_step delivers the observation tensor to host
 * memory; 1 by default), "zero_copy" (0/1, default 1: host-facing steps let the rasteriser store rows straight into the pinned host buffer, the
 * PCIe writes overlapping the drawing -- the HBM tensor is then stale and mv_obs_device refuses it until the next mv_step_device; 0:
 * rasterise into HBM in "host_slices" launches (0 = by size) whose downloads run on the copy engine while the next slice is drawn),
 * "fast_shading" (0/1, default 1: +-1 LSB fragment maths),
 * "tri_cap" (32..1022, default 368: the largest that leaves two CTAs per SM; triangles one raster CTA keeps in shared memory; a view with more is drawn in several batches,
 * results do not depend on it), "raster_bands" (row bands a view is cut into, one work item of the persistent raster grid each;
 * chosen from the number of views by default, results do not depend on it),
 * "raster_grid" (CTAs of the persistent raster grid, 0 = as many as the GPU holds (default): every raster launch of the engine -- the
 * step's frames, each slice of the sliced download, terminal frames, mv_draw_hires -- takes at most this many; engines that share one GPU
 * -- one per scenario of a mixed batch -- take a share each so that their grids run side by side instead of queueing behind each other;
 * results do not depend on it),
 * "raster_sched" (0/1/2, default 1: launches with more work items than raster CTAs draw the envs in the order of what their views cost in
 * the previous step, most expensive first, and the step kernel steps them in that order; 0 natural order, 2 always; results do not depend
 * on it),
 * "static_cap" (before the first reset: initial size of the per-level static-box arrays, default 768; they grow whenever a
 * generated level has more boxes -- the reference has no bound, component_voxel_grid.hpp:108-187),
 * "skip_unfit_levels" (0/1, default 0: a generated level that exceeds one of the remaining fixed capacities -- movable objects, reward
 * objects, terrain slabs, the dense grid -- makes mv_step / mv_reset fail with MV_ERR_CAPACITY, and keeps failing: the env would
 * otherwise leave the reference's level sequence; with 1 the env takes the next level of its stream instead and mv_levels_skipped
 * counts it),
 * "final_obs" (0/1, before the first reset, default 0: terminal frames of ended episodes, see mv_final_obs_host),
 * "segmentation" (0/1, before the first reset, default 0: the class and index of the drawable behind every pixel, see
 * mv_segmentation_host),
 * "state_tensors" (0/1, before the first reset, default 0: agent, env, object and reward rows beside the frames, see mv_state_tensors_host),
 * "action_repeat" (1..4, before the first reset (MV_ERR_STATE after it, MV_ERR_ARG outside the range), default 1: action repeat, or
 * frame skip, inside the engine.  Every step call (mv_step, mv_step_begin/end, mv_step_device[_ends]) runs up to k physics ticks of
 * 1/15 s per env with the same action masks, then draws once.  Interact acts on the first tick only (it toggles carrying, so one call
 * is one press); movement, look and jump repeat.  An episode end at tick j < k stops that env's ticks: it flips to its next level as
 * at any end, and the frame drawn is the new episode's first.  The reward of an agent is the float sum, in tick order from 0, of what
 * each tick paid; the tick that ends the episode pays 0, as a step that ends does.  Done, reason, true objective and terminal frame
 * are those of the ending tick.  Requested ends: see mv_step_device_ends.  k = 1 is the reference's step.  mv_reset, mv_reset_envs,
 * mv_states_load, mv_draw_hires and mv_debug_warp_agent run no ticks and are unchanged; state-store rows do not carry k.  The
 * cap: with k ticks per call and two level slots the asynchronous path needs episodes of 3k ticks, 0.8 s at k = 4 (DESIGN.md section 2);
 * option "level_slots" 4 lifts it),
 * "level_slots" (2 or 4, before the first reset (MV_ERR_STATE after it, MV_ERR_ARG for any other value), default 2: level slots per
 * env, one live and the rest holding the env's next levels in episode order.  With 2, mv_step_device[_ends] needs episodes of at least
 * three calls (see there).  With 4 it takes every episode length at every action_repeat k and honours every end request: an env ends
 * at most once per call, and the level replacing an end is on the device three calls later, when three ends have used the three staged
 * levels at most.  Outputs do not depend on it.  Cost of the two extra slots, in HBM and again in pinned host memory, per env: two
 * levels of 33 248 B, their static boxes (32 B each, static_cap of them) and rotations (8 B each), decorations (80 B each) and three
 * bit planes of the dense grid -- 374 KiB per Collect env (392 MB at 1 024 envs), 139 KiB per TowerBuilding env, 509 KiB per env of a
 * batch with an Obstacles env, plus 240 KiB per env for the hex mazes' decorations; state-store rows grow by the same.  The first
 * mv_reset generates three levels per env instead of one.  Ignored with option "level_set": nothing is staged),
 * "level_set" (L >= 0, before the first reset (MV_ERR_STATE after it), default 0 = off) and "level_set_seed" (s, default 0): train or
 * evaluate on a fixed set of levels, see "Level sets" below,
 * "overlap" (0/1, default 1: the raster kernel is a programmatic dependent launch of the step kernel and synchronises per env;
 * 0 serialises the kernels so that mv_last_kernel_ms can time them separately) */
int mv_set_option(mv_handle h, const char *key, int value);

/* Device-resident path (SURVEY.md 8f rank 1): the caller's consumer reads the tensors in HBM.
 * mv_step_device: like mv_step but takes the action masks from DEVICE memory (NULL = the engine's own buffer, see
 * mv_actions_device) and leaves the observation tensor on the device; rewards/dones still land on the host.  Contract: with two level
 * slots (the default) an env may end at most once in any three consecutive calls, else the call returns MV_ERR_STATE (see mv_sync); with
 * option "level_slots" 4 episodes of any length are accepted. */
int mv_step_device(mv_handle h, const int32_t *d_masks);
/* mv_step_device with per-env episode ends requested from the device: d_ends = uint8[num_envs] in DEVICE memory (NULL = none, which is
 * mv_step_device), read in the engine stream's order (mv_stream).  An env with d_ends[e] != 0 ends its episode at this step, after this
 * step's actions and scenario rules ran, exactly as a timer end: done = 1, reward 0, the true objective reported, flip to the pre-staged
 * next level, and the frame of this step is the new episode's first.  A request for an env whose current episode has run fewer than 3
 * steps (its step counter is below 3 after this step) is ignored: this call retires step k-2 at call k, so the next level of an env that
 * ended one or two steps ago is not staged yet.  The rule depends on the step count only, never on host timing.
 * With option "action_repeat" k the request applies after the call's last tick, and the rule reads "fewer than 3k ticks" (the tick
 * counter counts ticks, so it is still three calls).  A request for an env whose episode already ended at an earlier tick of the same
 * call is ignored: that end stands, with its own reason.  A call's reward is the sum of its ticks before the end.
 * With option "level_slots" 4 every request is honoured, including one in a new episode's first call: the next level is always staged. */
int mv_step_device_ends(mv_handle h, const int32_t *d_masks, const uint8_t *d_ends);
/* mv_step_device_ends with an active set (see mv_step_envs for what an inactive env does and reports): d_active = uint8[num_envs] in DEVICE
 * memory, read in the engine stream's order; non-zero means active.  d_active == NULL is mv_step_device_ends: the same kernels and launches. */
int mv_step_device_active(mv_handle h, const int32_t *d_masks, const uint8_t *d_ends, const uint8_t *d_active);
/* Restart chosen envs now: envs[i] start a new episode.  seeds == NULL: each continues its own level stream (it takes its pre-staged
 * next level, as at a natural episode end); else env envs[i] is first reseeded with seeds[i] and plays the first level of that stream --
 * it then behaves exactly as env envs[i] of a fresh engine after mv_seed_env and mv_reset (unlike mv_seed_env, a Sokoban env also drops
 * the rest of its shuffled level list, as a fresh engine has none).  Other envs are untouched.
 * Every view is drawn again and delivered as a step would (host buffer, HBM or mv_set_obs_buffer's, depth included; the other views
 * yield the same bytes); the restarted envs read reward 0 and done 0, as after mv_reset.  The episode counter keeps counting.
 * A synchronisation point like mv_states_load: it retires outstanding mv_step_device steps, and on return the restarted envs' levels after
 * next are generated and uploaded.  MV_ERR_ARG (n < 0, a null list with n > 0, an env out of range or listed twice) and MV_ERR_STATE
 * (before mv_reset, an outstanding mv_step_begin) change nothing; n == 0 does nothing.  Afterwards mv_last_kernel_ms gives [0] the
 * reset kernel and [1] the re-render. */
int mv_reset_envs(mv_handle h, const int32_t *envs, const int32_t *seeds, int n);
/* Redirect the HBM output of the rasteriser into caller-owned device memory: d_obs = uint8[N][h][w][4] (and d_depth = float[N][h][w]
 * when option depth is on; NULL keeps the engine's own).  Lets several engines -- one per scenario of a multi-task batch, reference
 * megaverse_env.py:27-39 -- write into slices of ONE contiguous tensor that a consumer or an NCCL gather reads without a staging copy.
 * NULL, NULL restores the engine's own buffers.  The pointer takes effect with the next step; steps already enqueued keep writing the
 * previous buffer (no synchronisation: a consumer that double-buffers its tensor -- e.g. to gather step t over NCCL while step t+1 is
 * drawn -- switches every step); mv_sync before freeing a buffer.  Steps with an active set (mv_step_device_active) draw every view into a
 * caller's buffer. */
int mv_set_obs_buffer(mv_handle h, uint8_t *d_obs, float *d_depth);
/* mv_step_device is ASYNCHRONOUS: it returns after enqueueing the step on the engine stream (device tensors are valid in
 * stream order).  mv_sync waits for everything enqueued and publishes the last step's rewards/dones/true objectives to the
 * host pointers.  Episode bookkeeping lags the device by two steps on this path, so with two level slots it needs episodes of at least
 * three steps (true with the scenarios' own parameters at action_repeat 1); a violation raises MV_FAULT_LEVEL_NOT_READY in mv_faults and
 * the next call returns MV_ERR_STATE.  Option "level_slots" 4 removes the limit. */
/* MegaverseGym::drawHires + getHiresObservation (megaverse.cpp:154-177,199-203): renders every agent view once more at w x h
 * (multiples of 32 x 4 up to 768 x 4096, e.g. the reference's 768 x 432: wider frames would take the window coordinates of the scenarios'
 * scenes past the range the rasteriser's integer set-up is exact in; mv_create takes the same width limit) from the state of the last step; *out = uint8[N][h][w][4], engine-owned,
 * valid until the next mv_draw_hires / mv_close */
int mv_draw_hires(mv_handle h, int w, int hgt, const uint8_t **out);
int mv_sync(mv_handle h);
/* Spectator cameras: draw chosen envs from caller-placed viewpoints with the step's rasteriser.  Camera c of n draws the instance list of env
 * envs[c] through the view matrix views16[c * 16 .. c * 16 + 16) (column-major, world to camera, the convention of mv_debug_get_view: the
 * camera looks down -z with y up; megaverse_b200/cameras.py builds them) into frame c: RGBA uint8[n][h][w][4], and on request view-space
 * depth float[n][h][w] and segmentation uint16[n][h][w] (MV_SEG_* << 8 | index).  The projection is the agents' at that size (100 degree
 * horizontal field of view); sizes follow mv_draw_hires: multiples of 32 x 4 up to 768 x 4096.  Neither option "depth" nor option
 * "segmentation" is needed.
 * Both calls draw the instance lists of the last completed step -- the state the observations show -- after active-set steps, restarts,
 * state loads, in mixed and level-set engines alike; camera c is drawn exactly as an agent view with the same matrix and size would be
 * (an agent's own matrix at the engine's size gives the step's frame, byte for byte, at 768 x 432 mv_draw_hires').  Neither call changes
 * any other output or any state a later step reads.
 * mv_draw_cameras: synchronous and host-facing.  envs and views16 are host tables; the frames land in engine-owned buffers (HBM and pinned
 * twins, grown on demand and kept: w * h * (4 + 4 + 2) B per camera each with depth and segmentation, 3.3 MB at 768 x 432), valid until the
 * next mv_draw_cameras or mv_close.  Any out pointer may be NULL; *depth / *seg are NULL when not requested.
 * mv_draw_cameras_device: asynchronous.  d_envs (int32[n]), d_views16 (float[n][16]) and the outputs (d_obs required, d_depth and d_seg
 * optional) are the caller's, in device memory.  Enqueued on the engine stream (mv_stream): between mv_step_device* calls it sees exactly
 * the state of the step before it; it does not drain the asynchronous ring.  An entry of d_envs outside [0, num_envs) draws an all-zero frame
 * (colour and alpha, depth, segmentation) and reads nothing.
 * Range counter: the integer set-up is exact while snapped window coordinates stay below 2^30.5 sub-pixels and corner differences below
 * 2^31.  Agent eyes stay inside by measurement; a caller-placed camera close to a large surface that crosses its camera plane far
 * off-axis may not.  Every camera launch counts the projected triangles (once per camera) that leave that range: a non-zero count means
 * some pixels of that launch may be wrong.  The host call returns it in *out_of_range; the device call gives in *d_out_of_range the
 * engine's uint32 counter, which holds the last camera launch's count in stream order.
 * Errors: MV_ERR_ARG for a null handle, n < 0, a null table (or, device call, a null d_obs) with n > 0, an env out of range in a host
 * table, a bad size; MV_ERR_STATE before mv_reset or with an mv_step_begin outstanding.  A rejected call changes nothing. */
int mv_draw_cameras(mv_handle h, const int32_t *envs, const float *views16, int n, int w, int hgt, int want_depth, int want_seg, const uint8_t **obs,
                    const float **depth, const uint16_t **seg, uint32_t *out_of_range);
int mv_draw_cameras_device(mv_handle h, const int32_t *d_envs, const float *d_views16, int n, int w, int hgt, uint8_t *d_obs, float *d_depth,
                           uint16_t *d_seg, uint32_t **d_out_of_range);
/* float[N][16] view matrices of the last step (view env*A + agent), in HBM, written by the step kernel in stream order: what chase cameras
 * are built from without leaving the device */
int mv_views_device(mv_handle h, float **d_views);
/* out6 = float[num_envs][6]: {min x, y, z, max x, y, z}, the world-space bounding box of each env's live level (static boxes, decorations,
 * terrain slabs), from the host mirrors: valid after host-facing calls and after mv_sync.  With a level set the bank row of the retired level
 * id.  MV_ERR_ARG for a null pointer, MV_ERR_STATE before mv_reset. */
int mv_level_bounds(mv_handle h, float *out6);
/* after mv_step_device steps: waits, then copies the device obs (and depth and segmentation, when enabled) into the host buffers that
 * mv_obs_host / mv_depth_host / mv_segmentation_host return */
int mv_fetch_obs(mv_handle h);
int mv_actions_device(mv_handle h, int32_t **d_masks);
int mv_obs_device(mv_handle h, uint8_t **d_obs);
int mv_depth_device(mv_handle h, float **d_depth);
int mv_rewards_device(mv_handle h, float **d_rewards);
int mv_dones_device(mv_handle h, uint8_t **d_dones);
/* uint8[num_envs] MV_END_* and float[N] true objectives of the last step in HBM, written by the step kernel in stream order */
int mv_done_reasons_device(mv_handle h, uint8_t **d_reasons);
int mv_true_objectives_device(mv_handle h, float **d_true_objectives);
/* the CUDA stream (cudaStream_t) all engine work is ordered on */
int mv_stream(mv_handle h, void **stream);

/* Level sets, option "level_set" L > 0 with option "level_set_seed" s (Procgen's num_levels / start_level).  The first mv_reset
 * generates, once, L levels for every distinct scenario name of the engine: level j of a scenario is the first level (episode 0) of a
 * fresh generator of that scenario seeded s + j with the engine's params -- what mv_debug_generate_level(scenario, A, s + j, 0, params)
 * dumps.  Generation runs on the worker pool; "skip_unfit_levels" and generation errors behave as for the streams.  The levels stay in
 * HBM as a bank of immutable rows that the envs share, and every env plays levels of its own scenario's rows only.  At each start of an
 * episode (a natural end, a requested end, mv_reset, mv_reset_envs) the step kernel chooses the env's next level j:
 *   1. the env's entry of the next-level array when it is in [0, L): used once, then set back to -1;
 *   2. else mv_level_set_pick(pick seed of the env, index of the new episode, L), a hash: uniform over the set, no state.
 * mv_seed, mv_seed_env and the seeds of mv_reset_envs set pick seeds (mv_seed: the value it would seed the env's generator with); they
 * never regenerate the bank, and the episode counter keeps counting.  Engines with the same options, seeds and actions play the same
 * level sequences and produce the same bytes.  A second mv_reset keeps the bank and starts every env on its next pick.
 * The host does nothing at an episode end, so mv_step_device[_ends|_active] takes every episode length at every action_repeat and honours
 * every end request (as with "level_slots" 4, which is ignored here), and mv_reset_envs waits for no generator.
 * Everything else is unchanged: frames, rewards, dones and reasons of an episode on level j equal those of a stream engine's episode on
 * the same level; final_obs, active sets, action repeat, segmentation, depth, mv_set_obs_buffer and mixed engines work as before.
 * State store: a row holds no level (the bank is the engine's): it carries the env's live row, pick seed and episode counter, so a
 * loaded or cloned env replays bit for bit, later levels included; mv_state_row_bytes shrinks by the level slabs.  The next-level array is
 * caller input like the actions and is not saved.
 * Memory (HBM, and again pinned for the host mirrors): one row per level and scenario, of 33 248 B + 40 B per static box (the capacity
 * is raised once to the largest level of the bank) + 80 B per decoration slot + three bit planes of the dense grid; DESIGN.md section 3
 * has the figures.  The per-env slot rings are not allocated.
 * mv_level_ids: host int32[num_envs], valid like mv_dones: the level each env is on after the last call -- for an env that just ended,
 *   the level of the NEW episode (the one the returned frame shows).  Inactive envs keep their value.  mv_level_ids_device: the same in
 *   HBM, written by the step kernel in stream order.
 * mv_next_levels_device: device int32[num_envs], engine-owned, initially -1 everywhere.  The caller writes it in the order of mv_stream
 *   (a prioritised-replay sampler's output, say).  The array is input from outside the engine: the kernel bounds every entry before use,
 *   and a value outside [0, L) is ignored (the engine picks) and left as it is.
 * mv_set_next_levels: the host form: entry envs[i] = levels[i], uploaded ahead of the next kernel.  MV_ERR_ARG for an env out of range or
 *   a level outside [0, L); nothing changes then.  Followed by mv_reset_envs(envs) it starts chosen envs on chosen levels now.
 * mv_level_set_pick: the hash itself (host-only, no handle), so that a caller can predict or verify a sequence.
 * The four calls with a handle return MV_ERR_STATE while "level_set" is 0. */
int mv_level_ids(mv_handle h, const int32_t **out);
int mv_level_ids_device(mv_handle h, int32_t **d_ids);
int mv_next_levels_device(mv_handle h, int32_t **d_next);
int mv_set_next_levels(mv_handle h, const int32_t *envs, const int32_t *levels, int n);
uint32_t mv_level_set_pick(uint32_t pick_seed, int32_t episode, int32_t count);

/* Env state store: save envs mid-episode and rewind or clone them later, on the device.  A store holds `rows` env states; a row is the
 * complete state of one env -- every per-env device array (env, agents, objects, object grid, instance list, views, both level slots,
 * rewards, dones, true objectives, fault bits) and the host state (the env's level generator and RNG, its live slot and episode index,
 * the host mirrors of both levels).  Reward shaping (it belongs to the agent index a policy sees), options, the engine-wide fault word
 * (mv_fault_word) and mv_levels_skipped stay with the engine.
 * mv_states_create: a store of `rows` rows, its id in *store; freed by mv_states_destroy or mv_close.
 * mv_states_save: copies env envs[i] into row rows[i] (rows distinct).
 * mv_states_load: env envs[i] continues exactly as the env saved into row rows[i] would have (same frames, rewards, dones and later
 * levels for the same actions); envs distinct, a row may go to several envs (clones run the same level stream).  Other envs are untouched.
 * A row loads only into an env of the saved env's scenario name (in a mixed engine, mv_create_mixed); otherwise the call is MV_ERR_ARG,
 * names both scenarios and changes nothing.
 * Afterwards every view is drawn again and delivered as a step would (host buffer, HBM or mv_set_obs_buffer's, depth included): the
 * loaded views show the frames of the saved step, and rewards / dones / true objectives read as they did after it.  A load is not an
 * episode end.
 * Save and load are synchronisation points: they retire outstanding mv_step_device steps and wait for the level generators.  Both need
 * mv_reset first and refuse an outstanding mv_step_begin (MV_ERR_STATE).  After either, mv_last_kernel_ms gives [0] the copy kernel
 * and [1] the re-render (0 after a save).  Stores belong to the engine that made them. */
int mv_states_create(mv_handle h, int rows, int *store);
int mv_states_save(mv_handle h, int store, const int32_t *envs, const int32_t *rows, int n);
int mv_states_load(mv_handle h, int store, const int32_t *rows, const int32_t *envs, int n);
int mv_states_destroy(mv_handle h, int store);
/* device bytes one row holds (grows with the static-box arrays, see option "static_cap"; without the level slabs with a level set) */
int mv_state_row_bytes(mv_handle h, int64_t *out);

/* sticky per-env fault bits ORed over all envs (MV_FAULT_* in mv_types.h); 0 = healthy */
int mv_faults(mv_handle h, int32_t *out);
/* the same bits without a device round trip: the step kernel ORs every fault it raises into a pinned host word (sticky).  Valid for
 * the steps whose results the host has (after mv_step / mv_step_end / mv_sync).  Non-zero means physics or level state left the
 * envelope the engine guarantees (MV_FAULT_* in csrc/mv_types.h): the Python MegaverseEnv raises on it. */
int mv_fault_word(mv_handle h, int32_t *out);
/* number of kernels the engine launched since creation */
int mv_kernel_launches(mv_handle h, int64_t *out);
/* device time of the last step's kernels in milliseconds: [0] step kernel, [1] raster kernel (CUDA events) */
int mv_last_kernel_ms(mv_handle h, float *out2);
/* device time of the last step's terminal-frame launch (option "final_obs") in milliseconds, CUDA events; 0 when the step had none or
 * carried no timing events (mv_step_device with option overlap 1).  With it, mv_last_kernel_ms [1] is the step's own raster launch. */
int mv_last_final_ms(mv_handle h, float *out);
/* device time of the last call's ray launches (mv_set_rays: the live rays and, with final_obs, the terminal ones) in milliseconds, CUDA
 * events; 0 when the call cast none or carried no timing events.  They run after the call's raster launches, and mv_last_kernel_ms and
 * mv_last_final_ms leave them out. */
int mv_last_rays_ms(mv_handle h, float *out);

/* MegaverseGym::close (megaverse.cpp:224-243) */
int mv_close(mv_handle h);

/* ---- introspection for parity tests (same layouts as the oracle's orc_get_* in oracle/orc_api.cpp) ---- */
int mv_debug_get_level(mv_handle h, int env, int32_t *out, int cap);
int mv_debug_get_state(mv_handle h, int env, float *out, int cap);
int mv_debug_get_voxels(mv_handle h, int env, int32_t *out, int cap);
int mv_debug_get_instances(mv_handle h, int env, float *out, int cap);
int mv_debug_get_view(mv_handle h, int env, int agent, float *out16);
/* test hook: put agent `agent` of env `env` somewhere else, as the character controller's warp does (the oracle's orc_scen_warp):
 * position pos[3] and basis9 (rows) are set, horizontal and vertical velocity become 0, nothing else changes.  The caller supplies all
 * twelve floats (e.g. read back from the oracle after its warp), so no rounding happens here.  Nothing is drawn: the next step renders
 * the warped agent.  A synchronisation point like mv_states_save: outstanding mv_step_device steps are retired first.  MV_ERR_STATE
 * before mv_reset or with an mv_step_begin outstanding; MV_ERR_ARG for an env or agent out of range, a null pointer or a non-finite
 * value.  On any error nothing changes. */
int mv_debug_warp_agent(mv_handle h, int env, int agent, const float pos[3], const float basis9[9]);
/* render caller-supplied instances (18 floats each: mesh, colour, 16 model) with one view matrix through the CUDA
 * rasteriser: rgba uint8[h][w][4], depth float[h][w] or NULL.  Host pointers.  Sizes with at most 128 tiles of 32 x 4; exact shading,
 * no segmentation, tri_cap 96, two row bands when the tile rows split evenly (else one): mv_debug_render_instances_ex with those options. */
int mv_debug_render_instances(const float *view16, const float *inst18, int n, int w, int h, uint8_t *rgba, float *depth);
/* The same with every variant of the raster kernel a step may launch.  opts[4] = {fast (0/1: the fast fragment stage of option
 * "fast_shading"), segmentation (0/1), tri_cap (0 = the engine default, else 32..1022), bands (0 = the rule of mv_draw_hires, about a
 * hundred 32 x 4 tiles per band; else 1..h/4 bands of equal height, the last one shorter)}.  Sizes as mv_draw_hires: multiples of 32 x 4
 * up to 768 x 4096; n <= 4096 instances sorted by mesh type, colours 0..21.  seg: uint16[h][w], required with segmentation 1: the tag of
 * each pixel's winner, instance i (0-based) drawn with tag i + 1, 0 where nothing was drawn.  stats: NULL or the kernel's 16 counters
 * (the ViewParams::stats layout: [4] clipped items, [5] triangles, [6] batches).  depth, seg and stats may be NULL.  MV_ERR_ARG for
 * a null view, instance, opts or rgba pointer or any value outside these ranges. */
int mv_debug_render_instances_ex(const float *view16, const float *inst18, int n, int w, int h, const int *opts, uint8_t *rgba, float *depth,
                                 uint16_t *seg, unsigned long long *stats);
/* Cast rays over caller-supplied scenes through the engine's ray launch (the one every drawing step enqueues): E envs of A agents in
 * one launch.  views16 = float[E*A][16] world-to-camera matrices; inst18 = float[E][stride][18] rows (mesh, colour, 16 model floats
 * column-major) and tags = int32[E][stride], the segmentation tag of each row (the rays skip the rows tagged MV_SEG_AGENT << 8 | agent
 * of the casting agent); counts = int32[E], the rows of each env cast against (the rest are not read); dirs3 = float[R][3] camera-space
 * directions, used as given; env_mask = uint8[E] or NULL: envs whose byte is 0 are not cast.  dist float[E*A][R] and tag uint16[E*A][R]
 * are in/out: uploaded first, so the rows of envs not cast come back as the caller filled them.  Host pointers; synchronous.
 * MV_ERR_ARG for a null pointer (env_mask apart), E outside 1..65536, A outside 1..MV_MAX_AGENTS, R outside 1..MV_MAX_RAYS, stride
 * outside 1..65536 or E * stride above 2^22, a count outside 0..stride, a cast row's mesh not one of 0..4, or max_dist not finite and
 * > 0; MV_ERR_CUDA when the device fails. */
int mv_debug_cast_rays(const float *views16, const float *inst18, const int32_t *tags, const int32_t *counts, int E, int A, int stride,
                       const float *dirs3, int R, float max_dist, const uint8_t *env_mask, float *dist, uint16_t *tag);
/* Run chosen contact cases through the step kernel's own collision code: the per-step candidate gather and culling envelope, then one
 * character-controller query, one warp per case (synchronous, host pointers).  A case is a collider set in collider order -- statics
 * [0, n_static_pre), the objects, statics [n_static_pre, n_static), the A agents' capsules -- and one query by agent `agent`.
 *   hdr8     int32[n][8]   {n_static_pre, n_static, n_obj, A, mode (0 sweep, 1 recover, 2 controller step), agent, 0, 0}
 *   boxes10  float[n][2 * MV_MAX_OBJECTS][10]  rows [0, n_static) the statics, rows MV_MAX_OBJECTS + [0, n_obj) the objects:
 *            centre[3], half extents[3], solid (statics) / enabled (objects) 0|1, rotated about Y 0|1 (statics only), local x axis (ax, az)
 *   agents3  float[n][MV_MAX_AGENTS][3]  capsule centres; the querying agent's own is where its envelope is centred (mode 2: the query's)
 *   query20  float[n][20]  sweep: from[3], to[3], filterDir[3], minSlopeDot; recover: point[3]; step: pos[3], hvel[3], vvel, voff, stepOff,
 *            jumpSpeed, jumpAxis[3], wasOnGround 0|1, wasJumping 0|1, dt > 0, maxSlopeCos
 * out_i8 int32[n][8] = {candidates, fault bits (MV_FAULT_CAND_OVERFLOW, MV_FAULT_ENVELOPE), hit / penetrated / wasOnGround, winning collider
 * index (-1 for none), winning feature (sweep: 0..22 for boxes, 0 for capsules; else -1), wasJumping, 0, 0}; out_f16 float[n][16] = sweep:
 * fraction, normal[3]; recover: delta[3]; step: pos[3], hvel[3], vvel, voff, stepOff, jumpSpeed; the rest 0.  MV_ERR_ARG, before any device
 * work, for a null pointer, n outside 1..65536, counts above MV_MAX_OBJECTS / MV_MAX_AGENTS, a bad mode or agent, a negative half
 * extent, a flag not 0 or 1, a rotated object, dt <= 0 or any non-finite float that the case uses; MV_ERR_CUDA when the device fails. */
int mv_debug_kcc(const int32_t *hdr8, const float *boxes10, const float *agents3, const float *query20, int n, int32_t *out_i8, float *out_f16);
/* host-only (no CUDA needed): run the level generator for the env RNG stream seeded with env_seed and dump the level of
 * episode `episode` (mv_debug_get_level layout, followed by each agent's 9 spawn-basis floats as bit patterns) */
int mv_debug_generate_level(const char *scenario, int num_agents, int env_seed, int episode, const char *const *param_keys,
                            const float *param_vals, int nparams, int32_t *out, int cap);
/* libstdc++ unordered_set iteration-order emulation (bzset.h): ops[i] = {op(0 insert,1 erase,2 clear), x, y, z};
 * writes the final iteration order as xyz triples, returns the element count */
/* per-env cycle stamps of the step kernel's phases: out = uint32[E][16] (0 staged, 1 actions, 2 candidate list, 3 controllers,
 * 4 transforms, 5 scenario, 6 outputs/reset, 7 instance list, 8 commit, 12 candidate count); enable=1 arms it, 0 frees it.  Stamps count
 * from the start of the call and cover the whole call: with option "action_repeat" 1..4 and 12 are those of the last tick it ran, 5 ends
 * the tick loop */
int mv_debug_step_profile(mv_handle h, uint32_t *out, int enable);
/* the cost-ordered raster queue as it stands (waits for the stream): the per-item costs of the last cost-ordered launch (N * H / 4 words,
 * N * bands of them used), the env order of the next one (num_envs words), the exit counter (one word).  Returns the number of words, or
 * minus that number when cap is smaller */
int mv_debug_view_order(mv_handle h, uint32_t *out, int cap);
/* rasteriser launch shape: out4 = {persistent grid size, CTAs per SM, dynamic shared memory per CTA in bytes, row bands per view} */
int mv_debug_raster_config(mv_handle h, int32_t *out4);
/* current size of the per-level static-box arrays (option "static_cap" at start, grows on demand) */
int mv_debug_static_cap(mv_handle h);
/* rasteriser work counters since the last enable: out16 = {work items, instances read, instances with visible items, items (box faces /
 * mesh triangles set up), items clipped at the near / far plane, triangles drawn, batches, -, then thread-0 cycle sums: head (work
 * claim, env stamp, view matrix), TMA waits, instance passes, item passes, final tile pass, whole work item, -, -}; enable=1 arms /
 * clears, 0 frees */
int mv_debug_raster_stats(mv_handle h, unsigned long long *out16, int enable);
/* host-only: colour tables of the generators + the rasteriser's palette (tests pin them against the reference's env/const.hpp) */
int mv_debug_color_tables(uint32_t *out, int cap);
/* host-only: default reward shaping ("R key=hexbits") and default float parameters ("P key=hexbits") of a scenario, one per line */
int mv_debug_defaults(const char *scenario, char *out, int cap);
/* host-only: number of levels among the first `episodes` of the env stream seeded env_seed that do not fit the engine's capacities */
int mv_debug_count_unfit_levels(const char *scenario, int num_agents, int env_seed, int episodes, const char *const *keys, const float *vals, int nparams);
/* levels replaced so far under option "skip_unfit_levels" (0 unless that option is set) */
int mv_levels_skipped(mv_handle h);
int mv_debug_bzset(const int32_t *ops, int nops, int32_t *out_xyz, int cap);

#ifdef __cplusplus
}
#endif
#endif
