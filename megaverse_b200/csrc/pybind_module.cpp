// pybind11 module `megaverse_b200.extension.megaverse`: the reference's MegaverseGym class surface
// (src/libs/bindings/megaverse.cpp:267-292 -- same method names, argument meaning and lifetime rules), implemented as a
// thin C++ host layer over the C ABI (include/megaverse_b200.h).  No CUDA or torch types cross this boundary.
//
// Differences that are deliberate and documented in INTEGRATION.md:
//   * use_vulkan is accepted and ignored: there is one backend (CUDA); without a GPU construction raises RuntimeError
//     (the reference would exit(-1) through TLOG(FATAL)).
//   * extra batched methods (set_actions_batch, get_observations, get_dones, ...) next to the per-agent ones, because the
//     reference's 2N+E+2 pybind round trips per step (SURVEY.md 3.2) would cap throughput far below the kernels.
//   * the GIL is released around reset()/step(), around states_save()/states_load() (env state store, not in the reference) and around
//     reset_envs() / step_envs() (restart chosen envs, step chosen envs; not in the reference).
//   * a second constructor takes a list of num_envs scenario names: a mixed-scenario batch in one engine (mv_create_mixed).
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <cctype>
#include <cstdlib>
#include <cstring>
#include <map>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

#include "megaverse_b200.h"

namespace py = pybind11;

namespace {

int g_logLevel = 2;
void setMegaverseLogLevel(int level) { g_logLevel = level; }  // tiny_logger.hpp:63-68; the engine itself does not log

class MegaverseGym {
public:
    MegaverseGym(const std::string &scenario, int w, int h, int numEnvs, int numAgentsPerEnv, int numSimulationThreads, bool useVulkan,
                 const std::map<std::string, float> &floatParams)
        : MegaverseGym(std::vector<std::string>(size_t(std::max(numEnvs, 0)), scenario), w, h, numEnvs, numAgentsPerEnv, numSimulationThreads, useVulkan, floatParams) {}
    // (extension) a mixed-scenario batch: env e runs scenarios[e] (mv_create_mixed)
    MegaverseGym(const std::vector<std::string> &scenarios, int w, int h, int numEnvs, int numAgentsPerEnv, int numSimulationThreads, bool useVulkan,
                 const std::map<std::string, float> &floatParams)
        : numEnvs_(numEnvs), numAgentsPerEnv_(numAgentsPerEnv), w_(w), h_(h) {
        (void)useVulkan;
        if (numEnvs > 0 && int(scenarios.size()) != numEnvs) throw std::invalid_argument("MegaverseGym: one scenario name per env expected");
        std::vector<const char *> names, keys;
        std::vector<float> vals;
        for (auto &s : scenarios) names.push_back(s.c_str());
        for (auto &kv : floatParams) { keys.push_back(kv.first.c_str()); vals.push_back(kv.second); }
        // the reference's constructor has no device argument (one process per GPU, CUDA_VISIBLE_DEVICES): MEGAVERSE_B200_DEVICE picks the
        // ordinal for processes that see several GPUs
        int device = 0;
        if (const char *dv = std::getenv("MEGAVERSE_B200_DEVICE")) device = std::atoi(dv);
        const int rc = mv_create_mixed(names.data(), w, h, numEnvs, numAgentsPerEnv, numSimulationThreads, device, keys.data(), vals.data(), int(keys.size()), &h__);
        if (rc != MV_OK) throw std::runtime_error(std::string("MegaverseGym: ") + mv_last_error(nullptr));
        masks_.assign(size_t(numEnvs) * numAgentsPerEnv, 0);
        std::set<std::string> distinct;  // level-set blocks: the engine keeps one per scenario, in any spelling
        for (auto s : scenarios) {
            for (char &c : s) c = char(std::tolower(static_cast<unsigned char>(c)));
            distinct.insert(s);
        }
        numBanks_ = int(distinct.size());
    }
    ~MegaverseGym() { close(); }

    void check(int rc) const {
        if (rc == MV_OK) return;
        const std::string msg = h__ ? mv_last_error(h__) : "closed";
        if (rc == MV_ERR_ARG) throw std::out_of_range(msg);
        throw std::runtime_error(msg);
    }
    void alive() const { if (!h__) throw std::runtime_error("MegaverseGym is closed"); }

    void seed(int seedValue) { alive(); check(mv_seed(h__, seedValue)); }
    int numAgents() const { return numAgentsPerEnv_; }
    std::vector<int> actionSpaceSizes() const { return {3, 3, 3, 2, 2, 3}; }  // Env::actionSpaceSizes, env.cpp:33

    void reset() {
        alive();
        int rc;
        { py::gil_scoped_release nogil; rc = mv_reset(h__); }
        check(rc);
    }
    void setActions(int envIdx, int agentIdx, std::vector<int> actions) {
        alive();
        if (envIdx < 0 || envIdx >= numEnvs_ || agentIdx < 0 || agentIdx >= numAgentsPerEnv_) throw std::out_of_range("set_actions: bad env/agent index");
        int32_t heads[6] = {0, 0, 0, 0, 0, 0};
        for (size_t i = 0; i < actions.size() && i < 6; ++i) heads[i] = actions[i];
        masks_[size_t(envIdx) * numAgentsPerEnv_ + agentIdx] = mv_encode_action(heads);
    }
    // batched extras: masks int32[N] (already encoded) or heads int32[N,6]
    void setActionsBatch(py::array_t<int32_t, py::array::c_style | py::array::forcecast> a) {
        alive();
        const size_t N = masks_.size();
        if (a.ndim() == 1 && size_t(a.shape(0)) == N) {
            std::memcpy(masks_.data(), a.data(), sizeof(int32_t) * N);
        } else if (a.ndim() == 2 && size_t(a.shape(0)) == N && a.shape(1) == 6) {
            for (size_t i = 0; i < N; ++i) masks_[i] = mv_encode_action(a.data() + i * 6);
        } else throw std::invalid_argument("set_actions_batch expects int32[N] masks or int32[N,6] heads");
    }
    void step() {
        alive();
        int rc;
        {
            py::gil_scoped_release nogil;
            rc = mv_set_actions(h__, masks_.data());
            if (rc == MV_OK) rc = mv_step(h__);
        }
        std::fill(masks_.begin(), masks_.end(), 0);  // env.cpp:140-142
        check(rc);
    }
    // (extension) step() of the listed envs only (mv_step_envs): the others run nothing, report reward 0 and not done, and keep their frames
    void stepEnvs(const std::vector<int32_t> &envs) {
        alive();
        int rc;
        {
            py::gil_scoped_release nogil;
            rc = mv_set_actions(h__, masks_.data());
            if (rc == MV_OK) rc = mv_step_envs(h__, envs.data(), int(envs.size()));
        }
        if (rc == MV_OK) std::fill(masks_.begin(), masks_.end(), 0);  // as after step(); a refused call changes nothing
        check(rc);
    }
    bool isDone(int envIdx) {
        alive();
        const uint8_t *d;
        check(mv_dones(h__, &d));
        if (envIdx < 0 || envIdx >= numEnvs_) throw std::out_of_range("is_done: bad env index");
        return d[envIdx] != 0;
    }
    std::vector<float> getLastRewards() {
        alive();
        const float *r;
        check(mv_rewards(h__, &r));
        return std::vector<float>(r, r + masks_.size());
    }
    py::array_t<uint8_t> getObservation(int envIdx, int agentIdx) {
        alive();
        const uint8_t *o;
        check(mv_obs_host(h__, &o));
        if (envIdx < 0 || envIdx >= numEnvs_ || agentIdx < 0 || agentIdx >= numAgentsPerEnv_) throw std::out_of_range("get_observation: bad env/agent index");
        const size_t view = size_t(envIdx) * numAgentsPerEnv_ + agentIdx;
        return py::array_t<uint8_t>({h_, w_, 4}, o + view * size_t(w_) * h_ * 4, py::none{});  // numpy object does not own memory
    }
    py::array_t<uint8_t> getObservations() {
        alive();
        const uint8_t *o;
        check(mv_obs_host(h__, &o));
        return py::array_t<uint8_t>({int(masks_.size()), h_, w_, 4}, o, py::none{});
    }
    py::array_t<float> getRewardsArray() {
        alive();
        const float *r;
        check(mv_rewards(h__, &r));
        return py::array_t<float>({int(masks_.size())}, r, py::none{});
    }
    py::array_t<uint8_t> getDones() {
        alive();
        const uint8_t *d;
        check(mv_dones(h__, &d));
        return py::array_t<uint8_t>({numEnvs_}, d, py::none{});
    }
    // (extension) why each env's episode ended at the last step: MV_END_* (0 not done, 1 time limit, 2 solved, 3 requested)
    py::array_t<uint8_t> getDoneReasons() {
        alive();
        const uint8_t *d;
        check(mv_done_reasons(h__, &d));
        return py::array_t<uint8_t>({numEnvs_}, d, py::none{});
    }
    // (extension) option "autoreset" 1 or 2: uint8[num_envs], 1 where the env's episode ended and its next one has not started
    py::array_t<uint8_t> getAwaitingReset() {
        alive();
        const uint8_t *d;
        check(mv_awaiting_reset_host(h__, &d));
        return py::array_t<uint8_t>({numEnvs_}, d, py::none{});
    }
    // (extension) terminal frames, option "final_obs": [N,h,w,4], the views of env e hold the frame its last episode ended on
    py::array_t<uint8_t> getFinalObservations() {
        alive();
        const uint8_t *o;
        check(mv_final_obs_host(h__, &o));
        return py::array_t<uint8_t>({int(masks_.size()), h_, w_, 4}, o, py::none{});
    }
    // (extension) option "segmentation": uint16 [N,h,w], MV_SEG_* class << 8 | index of the drawable behind each pixel, 0 where nothing was drawn
    py::array_t<uint16_t> getSegmentation() {
        alive();
        const uint16_t *o;
        check(mv_segmentation_host(h__, &o));
        return py::array_t<uint16_t>({int(masks_.size()), h_, w_}, o, py::none{});
    }
    py::array_t<float> getTrueObjectives() {
        alive();
        const float *t;
        check(mv_true_objectives(h__, &t));
        return py::array_t<float>({int(masks_.size())}, t, py::none{});
    }
    float trueObjective(int envIdx, int agentIdx) const {
        alive();
        const float *t;
        check(mv_true_objectives(h__, &t));
        if (envIdx < 0 || envIdx >= numEnvs_ || agentIdx < 0 || agentIdx >= numAgentsPerEnv_) throw std::out_of_range("true_objective: bad env/agent index");
        return t[size_t(envIdx) * numAgentsPerEnv_ + agentIdx];
    }
    // hi-res rendering (megaverse.cpp:148-177,199-203): the same rasteriser at renderW x renderH; the overview camera / viewer is
    // out of scope (a reference build without WITH_GUI does nothing there either)
    void setRenderResolution(int hiresW, int hiresH) { renderW_ = hiresW; renderH_ = hiresH; }
    void drawHires() {
        alive();
        py::gil_scoped_release nogil;
        check(mv_draw_hires(h__, renderW_, renderH_, &hires_));
    }
    void drawOverview() {}
    py::array_t<uint8_t> getHiresObservation(int envIdx, int agentIdx) {
        alive();
        if (!hires_) throw std::runtime_error("get_hires_observation before draw_hires");
        if (envIdx < 0 || envIdx >= numEnvs_ || agentIdx < 0 || agentIdx >= numAgentsPerEnv_) throw std::out_of_range("get_hires_observation: bad env/agent index");
        const size_t view = size_t(envIdx) * numAgentsPerEnv_ + agentIdx;
        return py::array_t<uint8_t>({renderH_, renderW_, 4}, hires_ + view * size_t(renderW_) * renderH_ * 4, py::none{});  // does not own memory
    }

    std::map<std::string, float> getRewardShaping(int envIdx, int agentIdx) {
        alive();
        const char *keys[32];
        float vals[32];
        int n = 0;
        check(mv_get_reward_shaping(h__, envIdx, agentIdx, keys, vals, 32, &n));
        std::map<std::string, float> m;
        for (int i = 0; i < n && i < 32; ++i) m[keys[i]] = vals[i];
        return m;
    }
    void setRewardShaping(int envIdx, int agentIdx, const std::map<std::string, float> &rs) {
        alive();
        std::vector<const char *> keys;
        std::vector<float> vals;
        for (auto &kv : rs) { keys.push_back(kv.first.c_str()); vals.push_back(kv.second); }
        check(mv_set_reward_shaping(h__, envIdx, agentIdx, keys.data(), vals.data(), int(keys.size())));
    }
    uintptr_t obsDevicePtr() { alive(); uint8_t *p; check(mv_obs_device(h__, &p)); return reinterpret_cast<uintptr_t>(p); }
    int faults() { alive(); int32_t f; check(mv_faults(h__, &f)); return f; }
    int faultWord() { alive(); int32_t f; check(mv_fault_word(h__, &f)); return f; }
    void setOption(const std::string &key, int value) {
        alive();
        check(mv_set_option(h__, key.c_str(), value));
        if (key == "level_set") levelSet_ = value;
    }
    int levelsSkipped() { alive(); return mv_levels_skipped(h__); }
    // env state store (include/megaverse_b200.h): save / load copy on the device and wait for it, so they run without the GIL
    int statesCreate(int rows) { alive(); int id = -1; check(mv_states_create(h__, rows, &id)); return id; }
    void statesSave(int store, const std::vector<int32_t> &envs, const std::vector<int32_t> &rows) {
        alive();
        if (envs.size() != rows.size()) throw std::invalid_argument("states_save: envs and rows differ in length");
        int rc;
        { py::gil_scoped_release nogil; rc = mv_states_save(h__, store, envs.data(), rows.data(), int(envs.size())); }
        check(rc);
    }
    void statesLoad(int store, const std::vector<int32_t> &rows, const std::vector<int32_t> &envs) {
        alive();
        if (envs.size() != rows.size()) throw std::invalid_argument("states_load: rows and envs differ in length");
        int rc;
        { py::gil_scoped_release nogil; rc = mv_states_load(h__, store, rows.data(), envs.data(), int(envs.size())); }
        check(rc);
    }
    void statesDestroy(int store) { alive(); check(mv_states_destroy(h__, store)); }
    // restart chosen envs now, optionally reseeded (mv_reset_envs); a synchronisation point like states_load, run without the GIL
    void resetEnvs(const std::vector<int32_t> &envs, std::optional<std::vector<int32_t>> seeds) {
        alive();
        if (seeds && seeds->size() != envs.size()) throw std::invalid_argument("reset_envs: envs and seeds differ in length");
        int rc;
        { py::gil_scoped_release nogil; rc = mv_reset_envs(h__, envs.data(), seeds ? seeds->data() : nullptr, int(envs.size())); }
        check(rc);
    }

    // (extension, option "level_set") the level of the set each env is on: for an env that just ended, the new episode's
    py::array_t<int32_t> getLevelIds() {
        alive();
        const int32_t *ids;
        check(mv_level_ids(h__, &ids));
        return py::array_t<int32_t>({numEnvs_}, ids, py::none{});
    }
    // (extension, option "state_tensors") {"agents": [N,16], "envs": [E,16], "objects": [E,128,4], "rewards": [E,128,4]}, views of the
    // engine's pinned rows (layout in the header); the terminal rows with option final_obs as well
    py::dict getStateTensors(bool terminal) {
        alive();
        const float *p[4];
        check(terminal ? mv_final_state_tensors_host(h__, &p[0], &p[1], &p[2], &p[3]) : mv_state_tensors_host(h__, &p[0], &p[1], &p[2], &p[3]));
        py::dict d;
        const int N = int(masks_.size());
        d["agents"] = py::array_t<float>({N, 16}, p[0], py::none{});
        d["envs"] = py::array_t<float>({numEnvs_, 16}, p[1], py::none{});
        d["objects"] = py::array_t<float>({numEnvs_, MV_STATE_OBJECT_ROWS, 4}, p[2], py::none{});
        d["rewards"] = py::array_t<float>({numEnvs_, MV_STATE_REWARD_ROWS, 4}, p[3], py::none{});
        return d;
    }
    // (extension, option "reward_components") float32 [N,8] views of the engine's pinned step rows, or episode rows (layout in the header)
    py::array_t<float> getRewardComponents(bool episode) {
        alive();
        const float *step, *ep;
        check(mv_reward_components_host(h__, &step, &ep));
        return py::array_t<float>({int(masks_.size()), int(MV_REWARD_COMPONENTS)}, episode ? ep : step, py::none{});
    }
    // (extension) ray sensors (mv_set_rays): directions float32 [R,3] in camera space, before the first reset
    void setRays(py::array_t<float, py::array::c_style | py::array::forcecast> dirs, float maxDist) {
        alive();
        if (dirs.size() % 3 != 0) throw std::invalid_argument("set_rays: directions must hold 3 floats per ray");
        const int n = int(dirs.size() / 3);
        check(mv_set_rays(h__, n ? dirs.data() : nullptr, n, maxDist));
        numRays_ = n;
    }
    // (dist float32 [N,R], tag uint16 [N,R]), views of the engine's pinned rays; the terminal rays with option final_obs as well
    py::tuple getRays(bool terminal) {
        alive();
        const float *d = nullptr;
        const uint16_t *t = nullptr;
        check(terminal ? mv_final_rays_host(h__, &d, &t) : mv_rays_host(h__, &d, &t));
        const int N = int(masks_.size());
        return py::make_tuple(py::array_t<float>({N, numRays_}, d, py::none{}), py::array_t<uint16_t>({N, numRays_}, t, py::none{}));
    }
    // (extension, option "level_set") bank row rows[i] (block * L + level) is to hold the first level of seed seeds[i] (mv_replace_levels)
    void replaceLevels(const std::vector<int32_t> &rows, const std::vector<int32_t> &seeds) {
        alive();
        if (rows.size() != seeds.size()) throw std::invalid_argument("replace_levels: rows and seeds differ in length");
        check(mv_replace_levels(h__, rows.data(), seeds.data(), int(rows.size())));
    }
    // (seeds int32 [B], retiring uint8 [B]) of the bank's rows (mv_level_rows), views valid like get_level_ids'
    py::tuple getLevelRows() {
        alive();
        const int32_t *seeds = nullptr;
        const uint8_t *retiring = nullptr;
        check(mv_level_rows(h__, &seeds, &retiring));
        const int B = levelSet_ * numBanks_;
        return py::make_tuple(py::array_t<int32_t>({B}, seeds, py::none{}), py::array_t<uint8_t>({B}, retiring, py::none{}));
    }
    void setNextLevels(const std::vector<int32_t> &envs, const std::vector<int32_t> &levels) {
        alive();
        if (envs.size() != levels.size()) throw std::invalid_argument("set_next_levels: envs and levels differ in length");
        check(mv_set_next_levels(h__, envs.data(), levels.data(), int(envs.size())));
    }

    // (extension) spectator cameras (mv_draw_cameras): camera c draws env envs[c] through the view matrix views[c] (float32 [n,16] or
    // [n,4,4] as stored, column-major) at w x h.  Returns (rgba uint8 [n,h,w,4], depth float32 [n,h,w] or None, seg uint16 [n,h,w] or None,
    // out-of-range triangle count), copies the caller keeps
    py::tuple drawCameras(const std::vector<int32_t> &envs, py::array_t<float, py::array::c_style | py::array::forcecast> views, int w, int h,
                          bool depth, bool seg) {
        alive();
        const int n = int(envs.size());
        if (views.size() != py::ssize_t(n) * 16) throw std::invalid_argument("draw_cameras: views must hold 16 floats per env");
        const uint8_t *o = nullptr;
        const float *d = nullptr;
        const uint16_t *sg = nullptr;
        uint32_t wide = 0;
        int rc;
        { py::gil_scoped_release nogil; rc = mv_draw_cameras(h__, envs.data(), views.data(), n, w, h, depth, seg, &o, &d, &sg, &wide); }
        check(rc);
        const size_t px = size_t(n) * size_t(w) * size_t(h);
        py::array_t<uint8_t> rgba({n, h, w, 4});
        if (px) std::memcpy(rgba.mutable_data(), o, px * 4);
        py::object dep = py::none(), sgo = py::none();
        if (depth) { py::array_t<float> a({n, h, w}); if (px) std::memcpy(a.mutable_data(), d, px * sizeof(float)); dep = a; }
        if (seg) { py::array_t<uint16_t> a({n, h, w}); if (px) std::memcpy(a.mutable_data(), sg, px * sizeof(uint16_t)); sgo = a; }
        return py::make_tuple(rgba, dep, sgo, wide);
    }
    // (extension) float32 [N,16] view matrices of the last step (mv_debug_get_view per view: waits for the stream)
    py::array_t<float> getViews() {
        alive();
        const int N = int(masks_.size());
        py::array_t<float> out({N, 16});
        for (int v = 0; v < N; ++v) check(mv_debug_get_view(h__, v / numAgentsPerEnv_, v % numAgentsPerEnv_, out.mutable_data() + size_t(v) * 16));
        return out;
    }
    // (extension) float32 [E,6] world-space bounding box {min xyz, max xyz} of each env's live level (mv_level_bounds)
    py::array_t<float> levelBounds() {
        alive();
        py::array_t<float> out({numEnvs_, 6});
        check(mv_level_bounds(h__, out.mutable_data()));
        return out;
    }

    void close() {
        if (h__) { mv_close(h__); h__ = nullptr; }
    }

private:
    mv_handle h__ = nullptr;
    int numEnvs_, numAgentsPerEnv_, w_, h_;
    int renderW_ = 768, renderH_ = 432;
    int numRays_ = 0;
    int numBanks_ = 1, levelSet_ = 0;
    const uint8_t *hires_ = nullptr;
    std::vector<int32_t> masks_;
};

}  // namespace

PYBIND11_MODULE(megaverse, m) {
    m.doc() = "megaverse_b200 Python bindings (MegaverseGym surface of the reference)";
    m.def("set_megaverse_log_level", &setMegaverseLogLevel, "Megaverse Log Level (0 to disable all logs, 2 for warnings");
    m.def(
        "reward_component_keys",
        [](const std::string &scenario) {
            const char *keys[MV_REWARD_COMPONENTS];
            if (mv_reward_component_keys(scenario.c_str(), keys) != MV_OK) throw std::invalid_argument("unknown scenario " + scenario);
            py::list out;
            for (const char *k : keys) out.append(k ? py::object(py::str(k)) : py::object(py::none()));
            return out;
        },
        py::arg("scenario"), "(extension) the shaping key of each reward-component column of a scenario, None for slot 0 and unused slots");
    py::class_<MegaverseGym>(m, "MegaverseGym")
        .def(py::init<const std::string &, int, int, int, int, int, bool, const std::map<std::string, float> &>())
        .def(py::init<const std::vector<std::string> &, int, int, int, int, int, bool, const std::map<std::string, float> &>())
        .def("num_agents", &MegaverseGym::numAgents)
        .def("action_space_sizes", &MegaverseGym::actionSpaceSizes)
        .def("seed", &MegaverseGym::seed)
        .def("reset", &MegaverseGym::reset)
        .def("set_actions", &MegaverseGym::setActions)
        .def("step", &MegaverseGym::step)
        .def("is_done", &MegaverseGym::isDone)
        .def("get_observation", &MegaverseGym::getObservation)
        .def("get_last_rewards", &MegaverseGym::getLastRewards)
        .def("true_objective", &MegaverseGym::trueObjective)
        .def("set_render_resolution", &MegaverseGym::setRenderResolution)
        .def("draw_hires", &MegaverseGym::drawHires)
        .def("draw_overview", &MegaverseGym::drawOverview)
        .def("get_hires_observation", &MegaverseGym::getHiresObservation)
        .def("get_reward_shaping", &MegaverseGym::getRewardShaping)
        .def("set_reward_shaping", &MegaverseGym::setRewardShaping)
        .def("close", &MegaverseGym::close)
        // batched / device extras
        .def("set_actions_batch", &MegaverseGym::setActionsBatch)
        .def("get_observations", &MegaverseGym::getObservations)
        .def("get_rewards", &MegaverseGym::getRewardsArray)
        .def("get_dones", &MegaverseGym::getDones)
        .def("get_true_objectives", &MegaverseGym::getTrueObjectives)
        .def("get_done_reasons", &MegaverseGym::getDoneReasons, "uint8[num_envs] why each episode ended at the last step: 0 not done, 1 time limit, 2 solved, 3 requested")
        .def("get_awaiting_reset", &MegaverseGym::getAwaitingReset, "uint8[num_envs] (option autoreset 1 or 2): 1 where the env's episode ended and its next one has not started")
        .def("get_final_observations", &MegaverseGym::getFinalObservations, "uint8[N,h,w,4] terminal frames (option final_obs): the frame each env's last episode ended on")
        .def("get_segmentation", &MegaverseGym::getSegmentation, "uint16[N,h,w] segmentation (option segmentation): class << 8 | index of the drawable behind each pixel, 0 where nothing was drawn")
        .def("obs_device_ptr", &MegaverseGym::obsDevicePtr)
        .def("faults", &MegaverseGym::faults)
        .def("fault_word", &MegaverseGym::faultWord)
        .def("set_option", &MegaverseGym::setOption)
        .def("levels_skipped", &MegaverseGym::levelsSkipped)
        .def("states_create", &MegaverseGym::statesCreate)
        .def("states_save", &MegaverseGym::statesSave)
        .def("states_load", &MegaverseGym::statesLoad)
        .def("states_destroy", &MegaverseGym::statesDestroy)
        .def("reset_envs", &MegaverseGym::resetEnvs, py::arg("envs"), py::arg("seeds") = py::none())
        .def("level_ids", &MegaverseGym::getLevelIds, "int32[num_envs] (option level_set): the level of the set each env is on; after an end, the new episode's")
        .def("set_next_levels", &MegaverseGym::setNextLevels, py::arg("envs"), py::arg("levels"),
             "(option level_set) env envs[i] plays level levels[i] in its next episode, once; followed by reset_envs(envs) it starts them on those levels now")
        .def("replace_levels", &MegaverseGym::replaceLevels, py::arg("rows"), py::arg("seeds"),
             "(option level_set) bank row rows[i] is to hold the first level of seed seeds[i]; it retires at the next call and is rewritten once no env is on it")
        .def("get_level_rows", &MegaverseGym::getLevelRows, "(option level_set) (seeds int32[B], retiring uint8[B]) of the bank's rows")
        .def("get_state_tensors", [](MegaverseGym &g) { return g.getStateTensors(false); },
             "dict of float32 views (option state_tensors): agents [N,16], envs [E,16], objects [E,128,4], rewards [E,128,4]")
        .def("set_rays", &MegaverseGym::setRays, py::arg("directions"), py::arg("max_distance"),
             "ray sensors, before the first reset: float32 [R,3] camera-space directions (x right, y up, -z forward), R in 0..256")
        .def("get_rays", [](MegaverseGym &g) { return g.getRays(false); },
             "(dist float32 [N,R], tag uint16 [N,R]): distance to the first front face along each ray (0: none) and its MV_SEG_* << 8 | index")
        .def("get_final_rays", [](MegaverseGym &g) { return g.getRays(true); },
             "the terminal rays (rays and option final_obs): cast from the scene each env's last episode ended on, same pair")
        .def("get_reward_components", [](MegaverseGym &g) { return g.getRewardComponents(false); },
             "float32 [N,8] view (option reward_components): the last call's reward split by the shaping slot that paid it")
        .def("get_episode_reward_components", [](MegaverseGym &g) { return g.getRewardComponents(true); },
             "float32 [N,8] view (option reward_components): the per-slot totals of each env's last finished episode")
        .def("get_final_state_tensors", [](MegaverseGym &g) { return g.getStateTensors(true); },
             "the terminal rows (options state_tensors and final_obs): the state each env's last episode ended on, same dict")
        .def("step_envs", &MegaverseGym::stepEnvs, py::arg("envs"),
             "step the listed envs only: the others run nothing, report reward 0 and done 0, and keep their observations")
        .def("draw_cameras", &MegaverseGym::drawCameras, py::arg("envs"), py::arg("views"), py::arg("w"), py::arg("h"), py::arg("depth") = false,
             py::arg("seg") = false,
             "spectator cameras: camera c draws env envs[c] through views[c] (16 floats, column-major) at w x h from the last step's scene; "
             "returns (rgba uint8[n,h,w,4], depth float32[n,h,w] or None, seg uint16[n,h,w] or None, out-of-range triangle count)")
        .def("get_views", &MegaverseGym::getViews, "float32[N,16] view matrices of the last step (view env*A + agent)")
        .def("level_bounds", &MegaverseGym::levelBounds, "float32[num_envs,6] {min xyz, max xyz} of each env's live level");
}
