// Host engine behind the C ABI (include/megaverse_b200.h): owns the HBM state, the host level generators and their
// worker pool, and launches the two kernels of a step on one CUDA stream.
//
//   mv_step  =  [H2D actions] -> stepKernel (physics + scenario + in-kernel reset + instance lists)
//                             -> viewKernel (geometry + raster + shading in shared memory -> obs tensor)
//                             -> [D2H obs/rewards/dones] -> schedule next-level generation
//
// There is no host synchronisation between physics, episode reset and rendering (the reference resets finished envs
// serially on the caller thread between the two, vector_env.cpp:94-105): every env always has its NEXT level pre-staged
// in HBM (no RNG draw happens during an episode, so the next level only depends on the env's RNG state after the
// previous generation), and the step kernel flips to it by itself when the episode ends.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <condition_variable>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <deque>
#include <functional>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <queue>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/megaverse_b200.h"
#include "hostmath.hpp"
#include "level_set.h"
#include "levelgen.hpp"
#include "raster_view.cuh"
#include "ray_kernel.h"
#include "state_copy.h"
#include "step_kernel.cuh"

namespace {

// every entry point runs on the engine's device and leaves the calling thread's current device as it found it
struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = (prev == dev) || cudaSetDevice(dev) == cudaSuccess;
        if (prev == dev) prev = -1;  // nothing to restore
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// the head of an entry point that takes a handle and touches the device: MV_ERR_ARG for a null handle, MV_ERR_CUDA when the switch to
// the engine's device fails, else the rest of the body runs on that device
#define MV_ON_DEVICE(h)                                                                                           \
    if (!(h)) return MV_ERR_ARG;                                                                                  \
    DeviceGuard dg__((h)->device);                                                                                \
    if (!dg__.ok) { (h)->setError("cudaSetDevice failed"); return MV_ERR_CUDA; }

thread_local std::string g_createError;

#define MV_CUDA(call)                                                                                             \
    do {                                                                                                          \
        cudaError_t err__ = (call);                                                                               \
        if (err__ != cudaSuccess) {                                                                               \
            setError(std::string(#call) + ": " + cudaGetErrorString(err__));                                      \
            return MV_ERR_CUDA;                                                                                   \
        }                                                                                                         \
    } while (0)

class WorkerPool {
public:
    explicit WorkerPool(int n) {
        for (int i = 0; i < n; ++i)
            threads_.emplace_back([this] {
                for (;;) {
                    std::function<void()> job;
                    {
                        std::unique_lock<std::mutex> lk(m_);
                        cv_.wait(lk, [this] { return stop_ || !q_.empty(); });
                        if (stop_ && q_.empty()) return;
                        job = std::move(q_.front());
                        q_.pop();
                    }
                    job();
                    {
                        std::lock_guard<std::mutex> lk(m_);
                        --pending_;
                    }
                    done_.notify_all();
                }
            });
    }
    ~WorkerPool() {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; }
        cv_.notify_all();
        for (auto &t : threads_) t.join();
    }
    void submit(std::function<void()> f) {
        { std::lock_guard<std::mutex> lk(m_); q_.push(std::move(f)); ++pending_; }
        cv_.notify_one();
    }
    void waitAll() {
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
    }

private:
    std::vector<std::thread> threads_;
    std::queue<std::function<void()>> q_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    int pending_ = 0;
    bool stop_ = false;
};

// The owners of the engine's CUDA resources.  Each releases what it holds when it is destroyed or given something else, and moves but
// never copies, so that every buffer, event and stream has exactly one owner.
//
// `count` elements of T in HBM (DevBuf) or in pinned host memory (PinBuf).  alloc first releases what the buffer holds and leaves it
// empty (p null, n 0) when it fails; free releases it early
template <typename T, bool Pinned> struct CudaBuf {
    T *p = nullptr;
    size_t n = 0;
    CudaBuf() = default;
    CudaBuf(const CudaBuf &) = delete;
    CudaBuf &operator=(const CudaBuf &) = delete;
    CudaBuf(CudaBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
    CudaBuf &operator=(CudaBuf &&o) noexcept {
        if (this != &o) { free(); p = std::exchange(o.p, nullptr); n = std::exchange(o.n, 0); }
        return *this;
    }
    ~CudaBuf() { free(); }
    cudaError_t alloc(size_t count) {
        free();
        void *q = nullptr;
        const size_t bytes = sizeof(T) * (count ? count : 1);
        const cudaError_t err = Pinned ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
        if (err == cudaSuccess) { p = static_cast<T *>(q); n = count; }
        return err;
    }
    void free() {
        if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); }
        p = nullptr; n = 0;
    }
};
template <typename T> using DevBuf = CudaBuf<T, false>;
template <typename T> using PinBuf = CudaBuf<T, true>;

// an event or a stream, created with flags; call sites take the raw handle through the conversion
template <typename H, cudaError_t (*Create)(H *, unsigned int), cudaError_t (*Destroy)(H)> struct CudaHandle {
    H h = nullptr;
    CudaHandle() = default;
    CudaHandle(const CudaHandle &) = delete;
    CudaHandle &operator=(const CudaHandle &) = delete;
    CudaHandle(CudaHandle &&o) noexcept : h(std::exchange(o.h, nullptr)) {}
    CudaHandle &operator=(CudaHandle &&o) noexcept {
        if (this != &o) { release(); h = std::exchange(o.h, nullptr); }
        return *this;
    }
    ~CudaHandle() { release(); }
    cudaError_t create(unsigned int flags) { release(); return Create(&h, flags); }
    operator H() const { return h; }

private:
    void release() { if (h) Destroy(h); h = nullptr; }
};
using CudaEvent = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using CudaStream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;

// an array of `rows` rows re-laid from a pitch of `from` elements to one of `to`: alloc() the new array, then apply() copies every row
// into it and moves it in.  A change allocates all of its arrays before it applies any, so that a failed allocation changes nothing
template <typename T, bool Pinned> struct Repitch {
    CudaBuf<T, Pinned> *buf; size_t rows, from, to; CudaBuf<T, Pinned> next{};
    bool alloc() { return next.alloc(rows * to) == cudaSuccess; }
    cudaError_t apply() {
        const cudaError_t err = cudaMemcpy2D(next.p, sizeof(T) * to, buf->p, sizeof(T) * from, sizeof(T) * from, rows, Pinned ? cudaMemcpyHostToHost : cudaMemcpyDeviceToDevice);
        if (err == cudaSuccess) *buf = std::move(next);
        return err;
    }
};

// The level arrays: rows in HBM with pinned mirrors, which the level workers write and the uploads, debug dumps and state stores read.  A
// row holds one MvLevel, staticCap static boxes and their 2 * staticCap rotation floats, decoCap decorations, and the solid, exit and lava
// bit planes of gridWords words each, of which its level uses levelWords[row].  Which env's level a row holds is the engine's to say.
struct LevelTable {
    int staticCap = MV_INITIAL_STATIC_CAP, decoCap = 0, gridWords = 0;  // the pitches; staticCap grows (growStatics)
    DevBuf<MvLevel> d_levels; DevBuf<MvBox> d_statics; DevBuf<float> d_staticRot; DevBuf<MvDeco> d_deco; DevBuf<uint32_t> d_solid;
    // `n` rows at the current pitches, on the device and pinned; a failure leaves every array empty
    bool alloc(size_t n) {
        const size_t cap = size_t(staticCap), deco = size_t(decoCap), w = size_t(gridWords) * 3;
        levelWords.assign(n, 0);
        if (d_levels.alloc(n) == cudaSuccess && d_statics.alloc(n * cap) == cudaSuccess && d_staticRot.alloc(n * cap * 2) == cudaSuccess &&
            d_deco.alloc(n * deco) == cudaSuccess && d_solid.alloc(n * w) == cudaSuccess && h_levels.alloc(n) == cudaSuccess &&
            h_statics.alloc(n * cap) == cudaSuccess && h_staticRot.alloc(n * cap * 2) == cudaSuccess && h_deco.alloc(n * deco) == cudaSuccess &&
            h_solid.alloc(n * w) == cudaSuccess)
            return true;
        d_levels.free(); d_statics.free(); d_staticRot.free(); d_deco.free(); d_solid.free();
        h_levels.free(); h_statics.free(); h_staticRot.free(); h_deco.free(); h_solid.free();
        return false;
    }
    // a level of at most staticCap static boxes into row r's mirrors, not uploaded.  Level workers write rows concurrently, never one row
    void write(size_t r, const mv::LevelOut &out) {
        std::memcpy(&h_levels.p[r], &out.level, sizeof(MvLevel));
        std::copy(out.statics.begin(), out.statics.end(), h_statics.p + r * size_t(staticCap));
        std::copy(out.staticRot.begin(), out.staticRot.end(), h_staticRot.p + r * size_t(staticCap) * 2);
        std::copy(out.deco.begin(), out.deco.end(), h_deco.p + r * size_t(decoCap));
        const size_t nw = std::min(out.solid.size(), size_t(gridWords));
        const std::vector<uint32_t> *planes[3] = {&out.solid, &out.exitBits, &out.lavaBits};
        for (int k = 0; k < 3; ++k) std::copy_n(planes[k]->begin(), nw, h_solid.p + (r * 3 + size_t(k)) * size_t(gridWords));
        levelWords[r] = int(nw);
    }
    // row r's mirrors as a level that write() puts back as it was (without the draw sequence, which only the generator reads)
    mv::LevelOut read(size_t r) const {
        const MvLevel &L = h_levels.p[r];
        const size_t ns = size_t(L.n_static), nd = size_t(std::max(0, L.n_deco)), nw = size_t(levelWords[r]);
        return {L, {statics(r), statics(r) + ns}, {rotations(r), rotations(r) + 2 * ns}, {deco(r), deco(r) + nd}, {},
                {plane(r, 0), plane(r, 0) + nw}, {plane(r, 1), plane(r, 1) + nw}, {plane(r, 2), plane(r, 2) + nw}};
    }
    // row r's mirrors into HBM on stream s: the level, its boxes and decorations, the words its planes use (Tower, Rearrange: one plane)
    cudaError_t upload(size_t r, cudaStream_t s) const {
        cudaError_t err = cudaSuccess;
        auto up = [&](void *dst, const void *src, size_t bytes) { if (err == cudaSuccess) err = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s); };
        const MvLevel &L = h_levels.p[r];
        up(&d_levels.p[r], &L, sizeof(MvLevel));
        if (L.n_static) {
            up(d_statics.p + r * size_t(staticCap), statics(r), sizeof(MvBox) * size_t(L.n_static));
            up(d_staticRot.p + r * size_t(staticCap) * 2, rotations(r), sizeof(float) * 2 * size_t(L.n_static));
        }
        if (L.n_deco > 0) up(d_deco.p + r * size_t(decoCap), deco(r), sizeof(MvDeco) * size_t(L.n_deco));
        const int planes = (L.scenario == MV_SCENARIO_TOWER || L.scenario == MV_SCENARIO_REARRANGE) ? 1 : 3;
        for (int k = 0; k < planes; ++k) up(d_solid.p + (r * 3 + size_t(k)) * size_t(gridWords), plane(r, k), sizeof(uint32_t) * size_t(levelWords[r]));
        return err;
    }
    // the static boxes and rotations at a pitch of `cap` boxes, device and pinned; no change unless every new array is allocated (else
    // cudaErrorMemoryAllocation) and filled
    cudaError_t growStatics(int cap) {
        const size_t rows = d_levels.n, was = size_t(staticCap), to = size_t(cap);
        Repitch<MvBox, false> d{&d_statics, rows, was, to};
        Repitch<float, false> dRot{&d_staticRot, rows, was * 2, to * 2};
        Repitch<MvBox, true> h{&h_statics, rows, was, to};
        Repitch<float, true> hRot{&h_staticRot, rows, was * 2, to * 2};
        if (!d.alloc() || !dRot.alloc() || !h.alloc() || !hRot.alloc()) return cudaErrorMemoryAllocation;
        cudaError_t err;
        if ((err = d.apply()) || (err = dRot.apply()) || (err = h.apply()) || (err = hRot.apply())) return err;
        staticCap = cap;
        return cudaSuccess;
    }
    // row views of the mirrors
    const MvLevel &level(size_t r) const { return h_levels.p[r]; }
    const MvBox *statics(size_t r) const { return h_statics.p + r * size_t(staticCap); }
    const float *rotations(size_t r) const { return h_staticRot.p + r * size_t(staticCap) * 2; }
    const MvDeco *deco(size_t r) const { return h_deco.p + r * size_t(decoCap); }
    const uint32_t *plane(size_t r, int k) const { return h_solid.p + (r * 3 + size_t(k)) * size_t(gridWords); }  // 0 solid, 1 exit, 2 lava

private:
    PinBuf<MvLevel> h_levels; PinBuf<MvBox> h_statics; PinBuf<float> h_staticRot; PinBuf<MvDeco> h_deco; PinBuf<uint32_t> h_solid;
    std::vector<int> levelWords;  // [rows] words of each bit plane the row's level uses
};

// one per-env device array as the state store sees it: `units` rows per env (the slot count for the arrays that hold the level slots, none
// of them with a level set) of unitBytes
struct EnvSlab {
    uint8_t *base;
    int units;
    size_t unitBytes;
    size_t rowBytes() const { return size_t(units) * unitBytes; }
};
constexpr int kSlabCount = 17;  // mv_engine::envSlabs()

// saved env states (mv_states_*): every per-env device row in arrays of `rows` rows with the engine's pitch, plus the host state
struct StateStore {
    int rows = 0;
    DevBuf<uint8_t> slabs[kSlabCount];  // same order as mv_engine::envSlabs()
    DevBuf<uint8_t> stateSlabs[4];      // option state_tensors: the live rows of the four state tensors (mv_engine::stateTensor order)
    DevBuf<uint8_t> rcSlabs[3];         // option reward_components: step rows, episode rows, running totals (mv_engine::rcTensor order)
    struct HostRow {
        bool saved = false;
        std::optional<mv::LevelGenerator> gen;  // the env's level stream; empty with a level set (the bank is the engine's, the pick is in MvEnvState)
        std::string scenario;                   // the saved env's scenario name: only an env of the same name may load the row
        int bankRow = -1, bankSeed = 0;         // level set: the bank row the env was on and the seed of the level it held then
        int slot = 0, episode = 0;
        std::vector<mv::LevelOut> levels;       // the level table's rows of the env's slots (option "level_slots"); none with a level set
    };
    std::vector<HostRow> host;
};

}  // namespace

static void fillConsts(MvConsts &k, int W, int H);
static_assert(MV_STATE_OBJECT_ROWS == MV_MAX_OBJECTS && MV_STATE_REWARD_ROWS == MV_MAX_REWARD, "state tensor rows");
static_assert(MV_REWARD_COMPONENTS == MV_R_COUNT, "reward component columns");

// the frame part of a raster launch: frame size, row bands of bandRows rows, the per-CTA spill slab (one band of the frame per CTA), the
// triangle-list capacity and the projection of k; the rest is zero (no stats, no ready stamps, no mask, natural order)
static mvr::ViewParams frameParams(int W, int H, int bands, int bandRows, unsigned long long *spill, int triCap, const MvConsts &k) {
    mvr::ViewParams vp = {};
    vp.W = W; vp.H = H; vp.bands = bands; vp.bandRows = bandRows; vp.spill = spill; vp.spillStride = W * bandRows; vp.triCap = triCap;
    vp.p00 = k.p00; vp.p11 = k.p11; vp.p22 = k.p22; vp.p32 = k.p32;
    return vp;
}

// Widest frame the rasteriser draws (mv_create, mv_draw_hires, the debug entries).  Its integer set-up -- int32 snapped positions and
// edge coefficients, int64 edge constants and bounds -- is exact while every snapped window coordinate |s| < 2^30.5 sub-pixels and every
// difference of two corners < 2^31 (tests/test_raster_conformance_gpu.py pins it; just beyond, the snap saturates or the coefficients wrap).
// A vertex the near clip makes lies on w = 0.01, so window coordinates grow with the lateral extent of the geometry crossing the camera
// plane, and with the frame's width only (the projection's y scale carries the aspect).  The scenarios' scenes reach |x_ndc| ~ 11 400 with
// corner differences ~ 17 400 (the hex mazes; tests/test_raster_independent.py measures them): at 768 wide |s| <= 2^30.06 and the
// differences <= 2^30.67; at 1024 the differences reach 2^31.08.
constexpr int kMaxRasterWidth = 768;
// triangle-list capacity of one raster CTA (shared memory) unless option tri_cap sets another; larger views are drawn in several batches
constexpr int kDefaultTriCap = 368;

// Frames drawn beside the step's own (mv_draw_hires, the camera launches, mv_debug_render_instances_ex's default): row bands of about a
// hundred 32x4 tiles each, so that a large frame keeps every CTA of the persistent grid busy
static int hiresBandRows(int w) { return std::max(1, 96 / (w / 32)) * 4; }
// the size rule of those frames: multiples of 32 x 4, at most kMaxRasterWidth x 4096
static bool hiresSizeOk(int w, int hgt) { return w >= 32 && hgt >= 4 && w % 32 == 0 && hgt % 4 == 0 && w <= kMaxRasterWidth && hgt <= 4096; }
// a device buffer of at least `count` elements, reallocated (contents lost) only when it is smaller
template <typename B> static cudaError_t ensureCapacity(B &b, size_t count) {
    if (b.p && b.n >= count) return cudaSuccess;
    b.free();
    return b.alloc(count);
}

// the raster kernel variant of a launch: the items it draws, whether it writes segmentation (never with terminal frames), the shading mode
using ViewKernel = void (*)(mvr::ViewParams);
static ViewKernel viewKernelOf(mvr::Items items, bool seg, bool fast) {
    using mvr::Items;
    using mvr::viewKernel;
    switch (items) {
    case Items::Ended: return fast ? viewKernel<true, Items::Ended> : viewKernel<false, Items::Ended>;
    case Items::Active:
        if (seg) return fast ? viewKernel<true, Items::Active, true> : viewKernel<false, Items::Active, true>;
        return fast ? viewKernel<true, Items::Active> : viewKernel<false, Items::Active>;
    case Items::Cameras:
        if (seg) return fast ? viewKernel<true, Items::Cameras, true> : viewKernel<false, Items::Cameras, true>;
        return fast ? viewKernel<true, Items::Cameras> : viewKernel<false, Items::Cameras>;
    default:
        if (seg) return fast ? viewKernel<true, Items::All, true> : viewKernel<false, Items::All, true>;
        return fast ? viewKernel<true> : viewKernel<false>;
    }
}

// the step kernel variant of a launch: level set, state tensors, reward components, autoreset mode
using StepKernel = void (*)(mvk::StepParams);
template <int kAuto> static StepKernel stepKernelOf(bool levelSet, bool state, bool rc) {
    using mvk::stepKernel;
    if (rc) {
        if (levelSet) return state ? stepKernel<true, true, true, kAuto> : stepKernel<true, false, true, kAuto>;
        return state ? stepKernel<false, true, true, kAuto> : stepKernel<false, false, true, kAuto>;
    }
    if (levelSet) return state ? stepKernel<true, true, false, kAuto> : stepKernel<true, false, false, kAuto>;
    return state ? stepKernel<false, true, false, kAuto> : stepKernel<false, false, false, kAuto>;
}
static StepKernel stepKernelOf(bool levelSet, bool state, bool rc, int autoreset) {
    return autoreset == 0 ? stepKernelOf<0>(levelSet, state, rc) : (autoreset == 1 ? stepKernelOf<1>(levelSet, state, rc) : stepKernelOf<2>(levelSet, state, rc));
}

struct mv_engine {
    std::string error;
    void setError(const std::string &e) { error = e; }

    int W = 0, H = 0, E = 0, A = 0, N = 0, threads = 1, device = 0;
    // every env runs its own scenario (mv_create_mixed); mv_create gives all envs the same one
    std::vector<std::string> envScenarioName;  // [E] the registered name the env was created with
    std::vector<int> envScenario;              // [E] MV_SCENARIO_* of that name
    std::vector<std::vector<std::pair<std::string, float>>> shaping;  // per agent view: ordered key list (std::map order)
    std::vector<mv::LevelGenerator> gens;
    std::mt19937 master{std::random_device{}()};
    std::unique_ptr<WorkerPool> pool;

    // pitch of the per-env grid arrays: the largest dense-grid capacity among the engine's scenarios (one pitch for all envs)
    int gridCells = 0;
    int triCap = kDefaultTriCap;
    std::atomic<int> maxObjSeen{0};
    bool wantDepth = false, obsToHost = true, didReset = false, fastShading = true;
    bool wantSeg = false;          // option "segmentation": the rasteriser also writes each pixel's drawable tag (d_seg / h_seg)
    bool hostStepPending = false;  // between mv_step_begin and mv_step_end
    bool skipUnfitLevels = false;  // option "skip_unfit_levels": replace a level that exceeds a fixed capacity by the stream's next one
    std::atomic<int> levelsSkipped{0};
    // host delivery of the obs tensor (host-facing steps).  zero copy (default): the raster kernel stores the rows straight into pinned
    // host memory, the PCIe writes overlap the drawing (measured best at 9 MB and at 151 MB per step on an H100: 45 GB/s effective at Collect 1024 x 4).
    // Otherwise: rasterise into HBM in host_slices launches, each slice's download on the copy engine while the next is drawn.
    int zeroCopyOpt = 1, hostSlicesOpt = 0;
    bool rasterToHost = false;
    bool deliverToHost = false;    // this launch's frames end up in the host buffers (zero copy, or a download behind the raster)
    bool deviceObsFresh = false;   // the HBM obs tensor holds the last step's frames (false after a zero-copy host-facing step)
    // A step with an active set draws only the active envs' views when its raster destination already holds every view's current frame:
    // the pinned host buffers (obs, depth, segmentation), or the engine's own HBM buffers -- never a caller's tensor (mv_set_obs_buffer),
    // whose rows the engine cannot vouch for.  Otherwise it draws every view.
    bool hostObsFresh = false, ownDeviceObsFresh = false;
    bool ownDeviceBuffers() const { return obsOut == d_obs.p && (!wantDepth || depthOut == d_depth.p); }
    int sliceCount = 1;            // this launch: > 1 = sliced download on copyStream
    CudaStream copyStream;
    std::vector<CudaEvent> sliceEv;
    int numSMs = 132;              // H100 SXM; replaced by the device's count in mv_create
    MvConsts consts{};

    CudaStream stream;
    // stream steps (mv_step_stream): the fork from the caller's stream onto the engine stream and the join back; stream mode from the
    // first one until mv_close (every other entry point is then a synchronisation point, see streamSync)
    CudaEvent evFork, evJoin;
    bool streamMode = false;
    // kernel times of the last timed call, read by readKernelTimes only.  The call records ev[0] before its first kernel, ev[1] after it
    // when its raster launch is serialised behind it, evFinal before a terminal-frame launch and ev[2] at the end
    CudaEvent ev[3];
    CudaEvent evFinal;
    enum class Timed { Union, Split, FirstOnly } timedAs = Timed::Union;  // no ev[1] (overlapping kernels), ev[1], no raster launch (a save)
    bool lastHadFinal = false;
    float lastMs[2] = {0, 0};
    float lastFinalMs = 0.0f;
    int64_t launches = 0;

    // Level slots (option "level_slots" D, 2 or 4): each env has one live slot and D - 1 staged ones that hold its next episodes' levels in
    // order; the step kernel moves to the next slot of the ring at an episode end.  Every [E][D] array below is laid out by it.
    int levelSlots = 2;
    // Level set (option "level_set" L > 0): the level arrays hold a bank instead, L levels per distinct scenario name of the engine, generated
    // once by the first reset and never written again.  Row bank * L + j is level j of scenario `bank`: episode 0 of a generator of that
    // scenario seeded levelSetSeed + j.  Envs share the rows: MvEnvState::slot is an env's live row, the step kernel chooses the next one
    // at an episode end (StepParams::levelSet), and the host does nothing per end.  "level_slots" is unused
    int levelSet = 0, levelSetSeed = 0;
    int numBanks = 1;                  // distinct scenario names among the envs
    std::vector<int> envBank;          // [E] which of them env e runs (in order of first appearance)
    std::vector<uint32_t> pickSeed;    // [E] the envs' pick seeds as last set by the host (MvEnvState::pad[0] is the live copy)
    DevBuf<int32_t> d_bankBase, d_levelIds, d_nextLevels;  // [E] each, see StepParams
    PinBuf<int32_t> h_levelIds;        // [E] level ids of the last retired call, beside h_dones
    PinBuf<int32_t> h_nextLevels;      // [E] staging of mv_set_next_levels
    // replaceable rows (mv_replace_levels, the header has the rule).  A request makes its row retiring from the next kernel-enqueuing call
    // on; the level is generated on replacePool into the request's own LevelOut meanwhile and copied into the row's mirrors and uploaded
    // only at the rewrite, at the start of the first call whose published level ids (those of call publishedCall) are at or after the
    // request's call and show no env on the row.  No device refcount is needed: from the request's kernel on no flip lands on the row, so
    // once a retired call shows it empty, no kernel still in flight can put an env back on it
    struct Replacement {
        int row = 0, seed = 0;
        int64_t call = -1;  // the call from whose kernel on the row is retiring (-1: requested since the last call)
        bool ready = false;
        std::string error;  // generation failed: reported by the rewrite call
        mv::LevelOut out;
    };
    std::vector<int32_t> rowSeed;      // [levelRows()] the seed of the level each row holds
    std::vector<uint8_t> rowRetiring;  // [levelRows()] a replacement of the row is pending
    std::vector<uint8_t> rowPickable;  // [levelRows()] what d_rowPickable holds (0 from a request's call to its rewrite)
    DevBuf<uint8_t> d_rowPickable;
    std::list<std::unique_ptr<Replacement>> replacements;  // pending, in request order
    std::unique_ptr<WorkerPool> replacePool;  // its own pool: the per-call flushUploads never waits for a replacement that is not due
    std::condition_variable replaceDone;      // with genMutex: a Replacement became ready
    int64_t stepCalls = 0;                    // kernel-enqueuing calls so far (mv_step*, mv_reset*)
    int64_t publishedCall = -1;               // the call whose level ids h_levelIds holds
    size_t levelRows() const { return levelSet ? size_t(levelSet) * size_t(numBanks) : size_t(E) * size_t(levelSlots); }
    // the row of the level arrays and their host mirrors that holds what MvEnvState::slot names for env e
    size_t rowOfSlot(int e, int slot) const { return levelSet ? size_t(slot) : size_t(e) * size_t(levelSlots) + size_t(slot); }
    // ... and the row of env e's live level as of the last retired call
    size_t liveRow(int e) const { return levelSet ? size_t(envBank[size_t(e)]) * size_t(levelSet) + size_t(h_levelIds.p[e]) : rowOfSlot(e, hostSlot[size_t(e)]); }
    LevelTable levels;             // [E][D] level slots, or the bank's rows; its static-box pitch grows with the levels (growStatics)
    DevBuf<uint8_t> d_objGrid;
    DevBuf<MvEnvState> d_envs;
    DevBuf<MvAgent> d_agents;
    DevBuf<MvObject> d_objects;
    DevBuf<MvInstance> d_inst;
    DevBuf<int32_t> d_instCounts;
    DevBuf<float> d_views;
    DevBuf<int32_t> d_actions;
    DevBuf<float> d_rtable;
    DevBuf<float> d_rewards;
    DevBuf<uint8_t> d_dones;
    DevBuf<uint8_t> d_doneReasons;  // [E] MV_END_* beside d_dones
    DevBuf<float> d_trueObj;
    DevBuf<uint8_t> d_obs;
    DevBuf<float> d_depth;
    DevBuf<uint16_t> d_seg;        // [N][H][W], with option segmentation (never redirected by mv_set_obs_buffer)
    uint8_t *obsOut = nullptr;     // where the rasteriser writes in HBM: d_obs, or the caller's tensor slice (mv_set_obs_buffer)
    float *depthOut = nullptr;
    DevBuf<int32_t> d_faults;
    // rasteriser (raster_view.cuh): a persistent grid of CTAs pulling (view, band) items from a counter that host-path calls never reset
    // (word E of d_ready, so that a stream step zeroes the stamps and the counter in one memset)
    uint32_t *workCounter() const { return d_ready.p + E; }
    uint32_t counterBase = 0;          // what the counter read before the next launch's first claim
    DevBuf<unsigned long long> d_spill;  // [rasterGrid][spillStride]
    DevBuf<unsigned long long> d_rasterStats;  // mv_debug_raster_stats only
    DevBuf<uint32_t> d_viewCost;       // cost-ordered work queue: [N * H / 4] cost per work item of the current raster launch (N * bands used), [E] env order for the next one, exit counter
    size_t costItems() const { return size_t(N) * size_t(H / 4); }
    int rasterGridCap = 0;             // option "raster_grid": upper bound of the raster grid (0: all CTAs the GPU holds) -- for several engines sharing one GPU
    int rasterSched = 1;               // option "raster_sched": 0 natural order, 1 cost-ordered when the launch has several items per CTA, 2 always
    int rasterGrid = 0, rasterCtasPerSM = 0, rasterBands = 1, bandRows = 0;
    size_t rasterSmem = 0;
    // hi-res pass (draw_hires): its own output buffers, allocated on first use
    struct Hires {
        int W = 0, H = 0;
        DevBuf<uint8_t> d_obs; PinBuf<uint8_t> h_obs;
        DevBuf<unsigned long long> spill;
    } hires;
    // camera launches (mv_draw_cameras[_device]): the host call's tables and output buffers, grown on demand and kept; the spill slab and
    // the out-of-range counter serve both calls
    struct Cameras {
        DevBuf<int32_t> d_env; DevBuf<float> d_views;
        DevBuf<uint8_t> d_obs; DevBuf<float> d_depth; DevBuf<uint16_t> d_seg;
        PinBuf<uint8_t> h_obs; PinBuf<float> h_depth; PinBuf<uint16_t> h_seg;
        DevBuf<unsigned long long> spill;
        DevBuf<uint32_t> d_range;  // [1] triangles of the last camera launch outside the integer set-up's exact range
        PinBuf<uint32_t> h_range;
    } cams;
    int cameraGrid = 0;  // persistent grid of the camera variants
    // pitch of the instance rows: the dynamic instances and every static box and decoration a level row can hold
    int instCap() const { return MV_DYN_INSTANCES + levels.staticCap + levels.decoCap; }

    // levels with more static boxes than the arrays hold: parked here by the workers until flushUploads has grown the arrays
    std::vector<std::pair<int, mv::LevelOut>> oversize;
    PinBuf<int32_t> h_actions;
    PinBuf<float> h_rtable;
    PinBuf<float> h_rewards;
    PinBuf<uint8_t> h_dones;
    PinBuf<uint8_t> h_doneReasons;
    PinBuf<float> h_trueObj;
    PinBuf<uint8_t> h_obs;
    PinBuf<float> h_depth;
    PinBuf<uint16_t> h_seg;
    PinBuf<int32_t> h_faults;
    PinBuf<int32_t> h_faultWord;   // OR of all fault bits raised so far, written by the step kernel (system-scope atomic)

    // mv_step_device pipeline: results of step k are consumed by the host while steps k+1, k+2 already run
    struct Pending { bool valid = false; uint64_t step = 0; int64_t call = 0; CudaEvent ev; PinBuf<float> rewards, trueObj; PinBuf<uint8_t> dones, reasons, awaiting; PinBuf<int32_t> levelIds; };
    std::vector<int64_t> lastAsyncDone;  // [E] asynchronous step index of the env's previous episode end
    bool asyncContractBroken = false;
    Pending ring[3];
    DevBuf<uint32_t> d_prof;  // mv_debug_step_profile only
    DevBuf<uint32_t> d_ready; // [E + 1]: per-env step completion stamps (step kernel -> geometry kernel), then the raster work counter
    uint32_t readyStamp = 0;  // the last host-path call's stamp: mv_reset's is 1, which every stream step uses (stepStream)
    bool overlap = true;      // geometry kernel launched as a programmatic dependent of the step kernel
    uint64_t asyncSteps = 0;

    std::vector<int> hostSlot, hostEpisode;   // mirrors of the device's live slot / episode index
    std::vector<int> pendingUpload;           // level ids (env * D + slot) whose freshly generated level waits for H2D
    // an env's levels come from one stateful generator (RNG stream, Sokoban's unplayed levels): its jobs run one after another, in the order
    // they were scheduled, on whichever worker drains the env's queue
    std::vector<std::deque<std::pair<int, int>>> genQueue;  // [E] (slot, serial) waiting for the env's generator
    std::vector<uint8_t> genBusy;                           // [E] a worker is draining the env's queue
    std::vector<std::string> genErrors;
    std::mutex genMutex;
    bool rtableDirty = true;

    std::vector<std::unique_ptr<StateStore>> stores;  // mv_states_create ids; null once destroyed
    PinBuf<int2> h_pairs;                              // (source row, destination row) of the last save / load
    DevBuf<int2> d_pairs;
    PinBuf<uint32_t> h_envList;                        // [E] the envs of the last mv_reset_envs
    DevBuf<uint32_t> d_envList;
    PinBuf<uint8_t> h_active;                          // [E] the active mask of the last mv_step_envs, uploaded to d_active
    DevBuf<uint8_t> d_active;

    // terminal frames (option "final_obs", allocated at the first reset): an env that ends in a step gets the frame that step would have
    // drawn had the episode not ended.  The step kernel writes the ending envs' terminal rows (instances at the pitch of d_inst, counts,
    // views); a masked raster launch over d_dones draws their views into the final-frame buffers: the pinned host ones for host-facing
    // steps, HBM for mv_step_device.  Rows of envs that did not end are never written.
    bool wantFinal = false;
    int actionRepeat = 1;           // option "action_repeat": physics ticks per step call (the step kernel's tick loop), drawn once
    bool finalOnDevice = false;    // the last terminal-frame launch stored into HBM (mv_fetch_obs copies the buffers down)
    int maskedGrid = 0;             // persistent grid of the masked raster variants (terminal frames, a step's active envs)
    DevBuf<MvInstance> d_termInst;  // [E][instCap]
    DevBuf<int32_t> d_termCounts;   // [E][8]
    DevBuf<float> d_termViews;      // [N][16]
    DevBuf<uint8_t> d_finalObs;     // [N][H][W][4]
    DevBuf<float> d_finalDepth;     // [N][H][W], with option depth
    PinBuf<uint8_t> h_finalObs;
    PinBuf<float> h_finalDepth;

    // autoreset (option "autoreset": 0 same-step, 1 next-step, 2 disabled).  Under 1 and 2 an ended env keeps its scene and is awaiting
    // (MvEnvState::pad[1]) until its flip; the step kernel writes every stepped env's flag into d_awaiting beside dones (and into the ring
    // slot's mirror), and the host keys its level bookkeeping on flips -- an env awaiting after the previous published call and not after
    // this one -- instead of on dones.  Nothing is allocated under 0
    int autoreset = 0;
    DevBuf<uint8_t> d_awaiting;            // [E]
    PinBuf<uint8_t> h_awaiting;            // [E] of the last published call, beside h_dones
    std::vector<uint8_t> awaitPrev, flips;  // [E] h_awaiting as the previous published call left it; this call's flips
    // the envs whose level bookkeeping advances with the call just published into h_dones / h_awaiting: the ended envs under same-step
    // autoreset, else the flips (a call that flips an env runs no tick for it, so it cannot also end it)
    const uint8_t *flipped() {
        if (!autoreset) return h_dones.p;
        for (int e = 0; e < E; ++e) flips[size_t(e)] = awaitPrev[size_t(e)] && !h_awaiting.p[e];
        noteAwaiting();
        return flips.data();
    }
    // a call that flips by itself (mv_reset, mv_reset_envs) or flips nothing (mv_states_load) was published: no flip to count
    void noteAwaiting() {
        if (autoreset) std::memcpy(awaitPrev.data(), h_awaiting.p, size_t(E));
    }

    // state tensors (option "state_tensors", allocated at the first reset): the step kernel writes every stepped env's rows (layout in the
    // header) into one HBM block, agents [N][16], envs [E][16], objects [E][MV_MAX_OBJECTS][4], rewards [E][MV_MAX_REWARD][4], followed
    // with option final_obs by the terminal rows in the same four shapes.  A host-facing call copies the whole block into its pinned twin
    // on copyStream while the frames are drawn; mv_step_device leaves it in HBM (mv_fetch_obs copies it down).
    bool wantState = false;
    bool stateCopyPending = false;  // this call's block download is on copyStream
    CudaEvent evState;              // the step kernel's rows are written: the download may start
    DevBuf<float> d_state;
    PinBuf<float> h_state;
    size_t stateFloats() const { return size_t(N) * 16 + size_t(E) * (16 + 4 * MV_MAX_OBJECTS + 4 * MV_MAX_REWARD); }
    size_t stateBlockFloats() const { return stateFloats() * (wantFinal ? 2 : 1); }
    // tensor k (0 agents, 1 envs, 2 objects, 3 rewards) of the live rows, or of the terminal rows
    float *stateTensor(float *block, int k, bool terminal) const {
        if (!block) return nullptr;
        const size_t off[4] = {0, size_t(N) * 16, size_t(N) * 16 + size_t(E) * 16, size_t(N) * 16 + size_t(E) * (16 + 4 * MV_MAX_OBJECTS)};
        return block + (terminal ? stateFloats() : 0) + off[k];
    }
    // bytes per env of tensor k (the state store's slabs)
    size_t stateRowBytes(int k) const {
        const size_t b[4] = {sizeof(float) * 16 * size_t(A), sizeof(float) * 16, sizeof(float) * 4 * MV_MAX_OBJECTS, sizeof(float) * 4 * MV_MAX_REWARD};
        return b[k];
    }
    // host-facing calls: the block into its pinned twin on copyStream, behind everything enqueued on the stream so far
    int downloadState() {
        if (!wantState) return MV_OK;
        MV_CUDA(cudaEventRecord(evState, stream));
        MV_CUDA(cudaStreamWaitEvent(copyStream, evState, 0));
        MV_CUDA(cudaMemcpyAsync(h_state.p, d_state.p, sizeof(float) * stateBlockFloats(), cudaMemcpyDeviceToHost, copyStream));
        stateCopyPending = true;
        return MV_OK;
    }

    // reward components (option "reward_components", allocated at the first reset): one HBM block of three [N][MV_R_COUNT] tensors -- the
    // step rows, the episode rows and the running totals of the episodes under way -- written by the step kernel (StepParams::rcStep).  A
    // host-facing call copies the first two into their pinned twin behind its step; mv_step_device leaves them in HBM (mv_fetch_obs
    // copies them down).  The running totals never leave the device
    bool wantRC = false;
    DevBuf<float> d_rc;
    PinBuf<float> h_rc;
    size_t rcFloats() const { return size_t(N) * MV_R_COUNT; }
    // tensor k (0 step rows, 1 episode rows, 2 running totals) of the block
    float *rcTensor(float *block, int k) const { return block ? block + size_t(k) * rcFloats() : nullptr; }
    size_t rcRowBytes() const { return sizeof(float) * MV_R_COUNT * size_t(A); }  // per env and tensor (the state store's slabs)
    int downloadRC(cudaStream_t s) {
        if (wantRC) MV_CUDA(cudaMemcpyAsync(h_rc.p, d_rc.p, sizeof(float) * 2 * rcFloats(), cudaMemcpyDeviceToHost, s));
        return MV_OK;
    }

    // ray sensors (mv_set_rays, allocated at the first reset): dist float[N][R] and tag uint16[N][R] in HBM, each followed with option
    // final_obs by the terminal rays of the same shape.  Every call that draws the step's frames casts them behind its raster launches
    // (castRays); a host-facing call then copies both blocks into their pinned twins on the stream
    int nRays = 0;
    float rayMaxDist = 0.0f;
    std::vector<float> rayDirs;     // [nRays][3] camera space, as the caller gave them
    DevBuf<float> d_rayDirs, d_rayDist;
    DevBuf<uint16_t> d_rayTag;
    PinBuf<float> h_rayDist;
    PinBuf<uint16_t> h_rayTag;
    CudaEvent evRays;               // before a timed call's ray launches (readKernelTimes)
    bool lastHadRays = false;
    float lastRaysMs = 0.0f;
    size_t rayCount() const { return size_t(N) * size_t(nRays); }
    size_t rayBlock() const { return rayCount() * (wantFinal ? 2 : 1); }
    // one ray launch: the live rays of the envs `mask` names (every env when null), or the terminal rays of the envs that ended (d_dones)
    // from their terminal rows
    int castRays(bool terminal, const uint8_t *mask) {
        mvray::RayParams rp;
        rp.instances = terminal ? d_termInst.p : d_inst.p; rp.instCounts = terminal ? d_termCounts.p : d_instCounts.p;
        rp.views = terminal ? d_termViews.p : d_views.p;
        rp.dirs = d_rayDirs.p; rp.envMask = terminal ? d_dones.p : mask;
        rp.dist = d_rayDist.p + (terminal ? rayCount() : 0); rp.tag = d_rayTag.p + (terminal ? rayCount() : 0);
        rp.instStride = instCap(); rp.E = E; rp.A = A; rp.R = nRays; rp.maxDist = rayMaxDist;
        MV_CUDA(mvray::castRays(rp, stream));
        launches += 1;
        return MV_OK;
    }
    // both blocks (live and terminal rays) into their pinned twins, in stream order
    int downloadRays(cudaStream_t s) {
        MV_CUDA(cudaMemcpyAsync(h_rayDist.p, d_rayDist.p, sizeof(float) * rayBlock(), cudaMemcpyDeviceToHost, s));
        MV_CUDA(cudaMemcpyAsync(h_rayTag.p, d_rayTag.p, sizeof(uint16_t) * rayBlock(), cudaMemcpyDeviceToHost, s));
        return MV_OK;
    }

    // ------------------------------------------------------------------ level generation scheduling
    // generate the level for episode `serial` of env e into staging slot s, after every job scheduled for the env before
    void scheduleGen(int e, int s, int serial) {
        {
            std::lock_guard<std::mutex> lk(genMutex);
            genQueue[size_t(e)].emplace_back(s, serial);
            if (genBusy[size_t(e)]) return;  // the worker draining the env's queue takes it next
            genBusy[size_t(e)] = 1;
        }
        pool->submit([this, e] {
            for (;;) {
                std::pair<int, int> job;
                {
                    std::lock_guard<std::mutex> lk(genMutex);
                    if (genQueue[size_t(e)].empty()) { genBusy[size_t(e)] = 0; return; }
                    job = genQueue[size_t(e)].front();
                    genQueue[size_t(e)].pop_front();
                }
                generateLevel(e, job.first, job.second);
            }
        });
    }
    // worker thread: one level of env e's stream into slot s
    void generateLevel(int e, int s, int serial) { generateInto(gens[size_t(e)], envScenario[size_t(e)], e * levelSlots + s, serial); }
    // worker thread: a bank level of MV_SCENARIO_* sc -- the first level of `gen` (a copy of the generator, as constructed, of an env of
    // that scenario) restarted with `seed`, which is what mv_debug_generate_level(..., seed, 0) dumps.  Into bank row `row`, or, for a
    // replacement, into its own LevelOut until the rewrite (the row's mirrors still hold the level live envs play)
    void generateBankLevel(mv::LevelGenerator gen, int sc, int row, int seed, Replacement *side = nullptr) {
        gen.restart((unsigned long)seed);
        if (!side) { generateInto(gen, sc, row, 0); return; }
        std::string error;
        generateOut(gen, sc, 0, side->out, &error);
        std::lock_guard<std::mutex> lk(genMutex);
        side->error = error;
        side->ready = true;
        replaceDone.notify_all();
    }
    // worker thread: the next level of `gen` (of MV_SCENARIO_* sc) into `out`; false on a generation error, which goes to *error when
    // given, else to genErrors
    bool generateOut(mv::LevelGenerator &gen, int sc, int serial, mv::LevelOut &out, std::string *error = nullptr) {
        // the env's own scenario's capacity, not the engine's pitch: a level is accepted exactly as in a single-scenario engine
        const int cap = mv::gridCapacity(sc);
        try {
            if (skipUnfitLevels) {
                const int skipped = gen.generateFitting(out, serial, cap);
                if (skipped) levelsSkipped.fetch_add(skipped);
            } else {
                gen.generate(out, serial, cap);
            }
        } catch (const std::exception &ex) {
            if (error) { *error = ex.what(); return false; }
            std::lock_guard<std::mutex> lk(genMutex);
            genErrors.push_back(ex.what());
            return false;
        }
        int curO = maxObjSeen.load();
        while (out.level.n_obj > curO && !maxObjSeen.compare_exchange_weak(curO, out.level.n_obj)) {}
        return true;
    }
    // worker thread: the next level of `gen` (of MV_SCENARIO_* sc) into row `id` of the level arrays
    void generateInto(mv::LevelGenerator &gen, int sc, int id, int serial) {
        mv::LevelOut out;
        if (!generateOut(gen, sc, serial, out)) return;
        if (int(out.statics.size()) > levels.staticCap) {  // the arrays are grown on the caller's thread (flushUploads), then the level goes in
            std::lock_guard<std::mutex> lk(genMutex);
            oversize.emplace_back(id, std::move(out));
            return;
        }
        stageLevel(id, out);
    }
    // worker thread (or flushUploads for parked levels): a generated level into its row's mirrors, and its upload queued
    void stageLevel(int id, const mv::LevelOut &out) {
        levels.write(size_t(id), out);
        std::lock_guard<std::mutex> lk(genMutex);
        pendingUpload.push_back(id);
    }
    // (re)allocate the level table ([E][D] slots, or the rows of a level set) and the instance rows, whose pitch depends on the table's
    int allocLevelSlots(const char *what) {
        if (!levels.alloc(levelRows()) || d_inst.alloc(size_t(E) * size_t(instCap())) != cudaSuccess) {
            setError(std::string(what) + ": allocation failed");
            return MV_ERR_CUDA;
        }
        return MV_OK;
    }
    // more static boxes per level: re-pitch every array that is laid out by the static-box pitch (level statics, instance lists)
    int growStatics(int need) {
        const int newCap = std::max(levels.staticCap * 2, ((need + 255) / 256) * 256);
        const int newInstCap = MV_DYN_INSTANCES + newCap + levels.decoCap;
        if (newInstCap > mvr::kMaxInstancesPerEnv) { setError("a level needs more drawables than the draw-order key can number"); return MV_ERR_CAPACITY; }
        MV_CUDA(cudaStreamSynchronize(stream));
        // the state stores keep the engine's pitch: every store slab whose unit grows is re-pitched alongside, over store rows x units rows
        Repitch<MvInstance, false> inst{&d_inst, size_t(E), size_t(instCap()), size_t(newInstCap)};
        std::vector<Repitch<uint8_t, false>> storeGrow;
        const auto was = envSlabs(), will = envSlabs(newCap, newInstCap);
        for (auto &st : stores)
            for (int k = 0; st && k < kSlabCount; ++k)
                if (will[size_t(k)].rowBytes() != was[size_t(k)].rowBytes())
                    storeGrow.push_back({&st->slabs[k], size_t(st->rows) * size_t(was[size_t(k)].units), was[size_t(k)].unitBytes, will[size_t(k)].unitBytes});
        bool ok = inst.alloc();
        for (auto &g : storeGrow) ok = ok && g.alloc();
        // the level table last: it changes only once its own arrays are allocated, and then every allocation has succeeded
        const cudaError_t err = ok ? levels.growStatics(newCap) : cudaErrorMemoryAllocation;
        if (err == cudaErrorMemoryAllocation) { setError("growing the static-box arrays: allocation failed"); return MV_ERR_CUDA; }
        MV_CUDA(err);
        MV_CUDA(inst.apply());
        for (auto &g : storeGrow) MV_CUDA(g.apply());
        if (d_termInst.p) {  // no copy: a terminal row is written whole before the launch that reads it
            if (d_termInst.alloc(size_t(E) * size_t(newInstCap)) != cudaSuccess) { setError("growing the terminal instance rows: allocation failed"); return MV_ERR_CUDA; }
        }
        return MV_OK;
    }
    int flushUploads() {
        pool->waitAll();
        std::vector<int> todo;
        {
            std::lock_guard<std::mutex> lk(genMutex);
            // sticky: the env whose level could not be generated would otherwise flip to a stale level later; only mv_close recovers
            if (!genErrors.empty()) { setError("level generation failed: " + genErrors.front()); return MV_ERR_CAPACITY; }
        }
        if (!oversize.empty()) {  // workers are idle (waitAll above): grow, then stage what they parked
            int need = 0;
            for (auto &po : oversize) need = std::max(need, int(po.second.statics.size()));
            const int rc = growStatics(need);
            if (rc) return rc;
            for (auto &po : oversize) stageLevel(po.first, po.second);
            oversize.clear();
        }
        {
            std::lock_guard<std::mutex> lk(genMutex);
            todo.swap(pendingUpload);
        }
        for (int id : todo) MV_CUDA(levels.upload(size_t(id), stream));
        return MV_OK;
    }

    void fillRtableRow(int view) {
        float *row = h_rtable.p + size_t(view) * MV_R_COUNT;
        for (int i = 0; i < MV_R_COUNT; ++i) row[i] = 0.0f;
        const int sc = envScenario[size_t(view / A)];
        for (auto &kv : shaping[size_t(view)]) {
            const int slot = mv::rewardSlot(sc, kv.first);
            if (slot >= 0) row[slot] = kv.second;
        }
    }

    mvk::StepParams stepParams(const int32_t *dActions, bool forceReset, Pending *mirror, const uint8_t *dEnds, const uint8_t *dActive = nullptr) {
        mvk::StepParams sp;
        sp.active = dActive;
        sp.hostRewards = mirror ? mirror->rewards.p : nullptr; sp.hostTrueObjectives = mirror ? mirror->trueObj.p : nullptr;
        sp.hostDones = mirror ? mirror->dones.p : nullptr;
        sp.hostFaults = h_faultWord.p;
        sp.levels = levels.d_levels.p; sp.statics = levels.d_statics.p; sp.staticRot = levels.d_staticRot.p; sp.staticCap = levels.staticCap; sp.solid = levels.d_solid.p;
        sp.objGrid = d_objGrid.p; sp.envs = d_envs.p; sp.agents = d_agents.p;
        sp.objects = d_objects.p; sp.instances = d_inst.p; sp.instCounts = d_instCounts.p; sp.views = d_views.p;
        sp.actions = dActions; sp.rtable = d_rtable.p; sp.rewards = d_rewards.p; sp.dones = d_dones.p; sp.trueObjectives = d_trueObj.p;
        sp.prof = d_prof.p;
        sp.deco = levels.d_deco.p; sp.decoCap = levels.decoCap; sp.instStride = instCap();
        sp.ready = d_ready.p; sp.readyStamp = ++readyStamp;
        sp.envOrder = rasterSched ? d_viewCost.p + costItems() : nullptr;  // a permutation at all times (identity until a cost-ordered raster launch has sorted it)
        sp.ends = dEnds;
        sp.repeat = actionRepeat;
        sp.slots = levelSlots;
        sp.levelSet = levelSet; sp.bankBase = d_bankBase.p; sp.nextLevels = d_nextLevels.p; sp.levelIds = d_levelIds.p;
        sp.hostLevelIds = (mirror && levelSet) ? mirror->levelIds.p : nullptr;
        sp.rowPickable = d_rowPickable.p;
        sp.doneReasons = d_doneReasons.p; sp.hostDoneReasons = mirror ? mirror->reasons.p : nullptr;
        sp.awaiting = autoreset ? d_awaiting.p : nullptr; sp.hostAwaiting = (autoreset && mirror) ? mirror->awaiting.p : nullptr;
        sp.termInstances = wantFinal ? d_termInst.p : nullptr; sp.termCounts = d_termCounts.p; sp.termViews = d_termViews.p;
        float *st = wantState ? d_state.p : nullptr, *termSt = wantFinal ? st : nullptr;
        sp.stAgents = stateTensor(st, 0, false); sp.stEnvs = stateTensor(st, 1, false); sp.stObjects = stateTensor(st, 2, false); sp.stRewards = stateTensor(st, 3, false);
        sp.termStAgents = stateTensor(termSt, 0, true); sp.termStEnvs = stateTensor(termSt, 1, true); sp.termStObjects = stateTensor(termSt, 2, true);
        sp.termStRewards = stateTensor(termSt, 3, true);
        float *rc = wantRC ? d_rc.p : nullptr;
        sp.rcStep = rcTensor(rc, 0); sp.rcEpisode = rcTensor(rc, 1); sp.rcRun = rcTensor(rc, 2);
        sp.maxObj = std::min(int(MV_MAX_OBJECTS), maxObjSeen.load());
        sp.E = E; sp.A = A; sp.gridCells = gridCells; sp.gridWords = levels.gridWords; sp.forceReset = forceReset ? 1 : 0;
        sp.k = consts;
        return sp;
    }
    // one warp per env of sp.E (sp.envOrder[w] when given)
    int launchStepKernel(const mvk::StepParams &sp) {
        const int warpsPerBlock = 2;
        const int blocks = (sp.E + warpsPerBlock - 1) / warpsPerBlock;
        const bool rc = sp.rcStep != nullptr;
        const size_t smem = (sizeof(mvk::WarpShared) + (rc ? mvk::kRcTickBytes : 0)) * warpsPerBlock;
        stepKernelOf(sp.levelSet > 0, sp.stAgents != nullptr, rc, autoreset)<<<blocks, warpsPerBlock * 32, smem, stream>>>(sp);
        MV_CUDA(cudaGetLastError());
        launches += 1;
        return MV_OK;
    }
    // One step (or forced flip) of sp.E envs: the step kernel, the raster launch of every view (of the active envs' views, see launchRaster,
    // when sp.active is set) -- a programmatic dependent of the step kernel when `dependent` and option overlap are on, else in stream order
    // behind it -- and, unless the step is a forced reset, the terminal frames of the envs that ended.  Every call but the asynchronous one
    // with option overlap records kernel times.  `capturable` (mv_step_stream): device work only -- results and terminal frames in HBM, no
    // event, no copy, and every view drawn (the host cannot vouch for the destination's rows at a graph replay)
    int launchStep(const mvk::StepParams &sp, bool dependent, bool capturable = false) {
        const bool async = sp.hostRewards != nullptr || capturable;  // mv_step_device: results land in its ring slot, terminal frames in HBM
        const bool dep = dependent && overlap, timed = !capturable && !(async && overlap), final = wantFinal && !sp.forceReset;
        if (timed) MV_CUDA(cudaEventRecord(ev[0], stream));
        if (const int rc = launchStepKernel(sp)) return rc;
        if (timed && !dep) MV_CUDA(cudaEventRecord(ev[1], stream));  // an event between the two kernels would serialise them
        // host-facing: the state block goes down while the frames are drawn -- or, behind a programmatic dependent raster launch, while its
        // terminal frames are (the event the download waits for would serialise the two kernels)
        if (!async && !dep) { if (const int rc = downloadState()) return rc; }
        if (const int rc = launchRaster(capturable ? nullptr : sp.active, dep ? sp.readyStamp : 0)) return rc;
        if (!async && dep) { if (const int rc = downloadState()) return rc; }
        if (final) {  // after the step's own frames: the terminal frames of the envs that ended (stream order, no stamps)
            if (timed) MV_CUDA(cudaEventRecord(evFinal, stream));
            if (const int rc = launchFinal(!async)) return rc;
        }
        if (nRays) {  // behind every raster launch of the call: the rays of the stepped envs, then the terminal rays of those that ended
            if (timed) MV_CUDA(cudaEventRecord(evRays, stream));
            if (const int rc = castRays(false, sp.active)) return rc;
            if (final) { if (const int rc = castRays(true, nullptr)) return rc; }
        }
        if (const int rc = endTimes(dep ? Timed::Union : Timed::Split, timed, final, nRays > 0)) return rc;
        return (nRays && !async) ? downloadRays(stream) : MV_OK;
    }
    // the last event of a call (ev[2], only when `timed`) and what its events bracket, for readKernelTimes
    int endTimes(Timed kind, bool timed = true, bool hadFinal = false, bool hadRays = false) {
        if (timed) MV_CUDA(cudaEventRecord(ev[2], stream));
        timedAs = kind;
        lastHadFinal = timed && hadFinal;
        lastHadRays = timed && hadRays;
        return MV_OK;
    }
    // the masked raster launch over the terminal rows: every (view, band) item of an env whose d_dones byte is set, into the final-frame
    // buffers -- pinned host memory (stored through UVA, like the zero-copy obs rows) or HBM
    int launchFinal(bool toHost) {
        mvr::ViewParams vp = frameParams(W, H, rasterBands, bandRows, d_spill.p, triCap, consts);
        vp.instances = d_termInst.p; vp.instCounts = d_termCounts.p; vp.views = d_termViews.p;
        vp.obs = toHost ? h_finalObs.p : d_finalObs.p; vp.depth = wantDepth ? (toHost ? h_finalDepth.p : d_finalDepth.p) : nullptr;
        vp.viewBase = 0; vp.N = N;
        vp.envMask = d_dones.p;
        finalOnDevice = !toHost;
        return launchView(vp, false, mvr::Items::Ended);
    }
    // CTAs of a launch: the persistent grid of the kernel variant, at most option raster_grid, at most one per work item
    int rasterGridFor(const mvr::ViewParams &vp) const {
        const int full = vp.camEnv ? cameraGrid : (vp.envMask ? maskedGrid : rasterGrid);
        return std::min(rasterGridCap > 0 ? std::min(full, rasterGridCap) : full, vp.N * vp.bands);
    }
    // One persistent launch over all (view, band) items.  Every CTA makes exactly one failing claim when the queue is empty, so the
    // work counter advances by items + grid per launch and the host keeps the base instead of resetting the counter (no memset node
    // between the step kernel and its programmatic dependent).  Every engine launch reads instance lists at the engine's pitch.
    int launchView(mvr::ViewParams &vp, bool dependent, mvr::Items items = mvr::Items::All) {
        const int grid = rasterGridFor(vp);
        vp.A = A; vp.instStride = instCap();
        vp.workCounter = workCounter(); vp.counterBase = counterBase;
        counterBase += uint32_t(vp.N) * uint32_t(vp.bands) + uint32_t(grid);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(unsigned(grid)); cfg.blockDim = dim3(mvr::kThreads); cfg.dynamicSmemBytes = rasterSmem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = dependent ? 1 : 0;
        MV_CUDA(cudaLaunchKernelEx(&cfg, viewKernelOf(items, vp.seg != nullptr, fastShading), vp));
        launches += 1;
        return MV_OK;
    }
    // the cost-ordered queue starts in natural order
    cudaError_t resetViewOrder() {
        std::vector<uint32_t> init(costItems() + size_t(E) + 1, 0u);  // item costs, env order, exit counter
        for (int e = 0; e < E; ++e) init[costItems() + size_t(e)] = uint32_t(e);
        return cudaMemcpy(d_viewCost.p, init.data(), sizeof(uint32_t) * init.size(), cudaMemcpyHostToDevice);
    }
    // depStamp: the ready stamp of the step kernel just enqueued when this is its programmatic dependent launch, else 0.  active: the step's
    // active mask (or nullptr): when the destination already holds every view's current frame, only the views of the active envs are drawn
    // -- the rows of the others stay
    int launchRaster(const uint8_t *active, uint32_t depStamp) {
        const bool dep = depStamp != 0;
        mvr::ViewParams vp = frameParams(W, H, rasterBands, bandRows, d_spill.p, triCap, consts);
        vp.instances = d_inst.p; vp.instCounts = d_instCounts.p; vp.views = d_views.p;
        // pinned allocations are mapped into the device address space (UVA), so the kernel can store through the host pointer
        vp.obs = rasterToHost ? h_obs.p : obsOut; vp.depth = wantDepth ? (rasterToHost ? h_depth.p : depthOut) : nullptr;
        vp.seg = wantSeg ? (rasterToHost ? h_seg.p : d_seg.p) : nullptr;
        vp.stats = d_rasterStats.p;
        // programmatic dependent launch: the grid may start before the step kernel has drained; a CTA waits for its env's stamp
        vp.ready = dep ? d_ready.p : nullptr; vp.readyStamp = depStamp;
        const bool fresh = rasterToHost ? hostObsFresh : (ownDeviceObsFresh && ownDeviceBuffers());
        const uint8_t *mask = fresh ? active : nullptr;
        const mvr::Items items = mask ? mvr::Items::Active : mvr::Items::All;
        vp.envMask = mask;
        deviceObsFresh = !rasterToHost;
        ownDeviceObsFresh = !rasterToHost && ownDeviceBuffers();
        hostObsFresh = deliverToHost;
        if (sliceCount <= 1) {
            vp.viewBase = 0; vp.N = N;
            if (rasterSched == 2 || (rasterSched == 1 && N * rasterBands > rasterGridFor(vp))) {  // more work items than CTAs: their order matters
                vp.viewCost = d_viewCost.p; vp.order = d_viewCost.p + costItems(); vp.exitCounter = d_viewCost.p + costItems() + size_t(E);
            }
            return launchView(vp, dep, items);
        }
        // sliced download: whole envs per slice; slice s is copied down by the copy engine while slice s+1 is rasterised (whole slices also
        // with an active mask: their rows are current either way)
        const int perSlice = ((E + sliceCount - 1) / sliceCount) * A;
        for (int base = 0, si = 0; base < N; base += perSlice, ++si) {
            const int cnt = std::min(perSlice, N - base);
            vp.viewBase = base; vp.N = cnt;
            vp.envMask = mask ? mask + base / A : nullptr;
            const int rc = launchView(vp, dep && si == 0, items);
            if (rc) return rc;
            while (int(sliceEv.size()) <= si) { CudaEvent e2; MV_CUDA(e2.create(cudaEventDisableTiming)); sliceEv.push_back(std::move(e2)); }
            MV_CUDA(cudaEventRecord(sliceEv[size_t(si)], stream));
            MV_CUDA(cudaStreamWaitEvent(copyStream, sliceEv[size_t(si)], 0));
            if (const int rcd = downloadViews(base, cnt, copyStream)) return rcd;
        }
        return MV_OK;
    }
    // views [base, base + cnt) of the HBM frames -- obs, and depth and segmentation when they are on -- into the host buffers
    int downloadViews(int base, int cnt, cudaStream_t s) {
        const size_t px = size_t(W) * H, off = size_t(base) * px, n = size_t(cnt) * px;
        MV_CUDA(cudaMemcpyAsync(h_obs.p + off * 4, obsOut + off * 4, n * 4, cudaMemcpyDeviceToHost, s));
        if (wantDepth) MV_CUDA(cudaMemcpyAsync(h_depth.p + off, depthOut + off, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
        if (wantSeg) MV_CUDA(cudaMemcpyAsync(h_seg.p + off, d_seg.p + off, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost, s));
        return MV_OK;
    }
    // decide how this host-facing launch delivers its frames: zero-copy stores, or into HBM and then one copy (sliceCount 1) or a
    // download per slice of whole envs (sliceCount > 1)
    void chooseDelivery(bool copyObs) {
        deliverToHost = copyObs;
        rasterToHost = copyObs && zeroCopyOpt != 0;
        if (!copyObs || rasterToHost) sliceCount = 1;
        else if (hostSlicesOpt > 0) sliceCount = std::min(hostSlicesOpt, E);
        else {  // four slices: the best copy-engine form at 151 MB (H100)
            const size_t bytes = size_t(N) * W * H * ((wantDepth ? 8 : 4) + (wantSeg ? 2 : 0));
            sliceCount = int(std::max<size_t>(1, std::min<size_t>({size_t(4), size_t(E), bytes / (size_t(32) << 20)})));
        }
    }
    // draw_hires (megaverse.cpp:154-177): every agent view once more, at (w, h), from the instance lists and camera matrices of
    // the last step -- the same kernel over row bands of the large frame.  Result in hires.h_obs, uint8[N][h][w][4].
    int drawHires(int w, int hgt) {
        if (!didReset) { setError("mv_draw_hires before mv_reset"); return MV_ERR_STATE; }
        if (!hiresSizeOk(w, hgt)) {
            setError("hi-res size must be a multiple of 32 x 4, at most 768 x 4096");
            return MV_ERR_ARG;
        }
        int rc = drain();
        if (rc) return rc;
        if (hires.W != w || hires.H != hgt) {
            hires = {};  // the old size's buffers go before the new ones are allocated
            const size_t px = size_t(N) * w * hgt * 4;
            if (hires.d_obs.alloc(px) != cudaSuccess || hires.h_obs.alloc(px) != cudaSuccess) {
                setError("hi-res buffers: allocation failed");
                return MV_ERR_CUDA;
            }
            hires.W = w; hires.H = hgt;
        }
        mvr::ViewParams vp;
        rc = bandedFrame(w, hgt, rasterGrid, hires.spill, vp);
        if (rc) return rc;
        vp.instances = d_inst.p; vp.instCounts = d_instCounts.p; vp.views = d_views.p;
        vp.obs = hires.d_obs.p;
        vp.viewBase = 0; vp.N = N;
        rc = launchView(vp, false);
        if (rc) return rc;
        MV_CUDA(cudaMemcpyAsync(hires.h_obs.p, hires.d_obs.p, size_t(N) * w * hgt * 4, cudaMemcpyDeviceToHost, stream));
        MV_CUDA(cudaStreamSynchronize(stream));
        return MV_OK;
    }
    // The frame part of a launch at w x h beside the step's own (mv_draw_hires, cameras) by a grid of `grid` CTAs: the hi-res band rule,
    // the projection of that size, and a spill slab of one band per CTA in `spill` (grown when it is too small)
    int bandedFrame(int w, int hgt, int grid, DevBuf<unsigned long long> &spill, mvr::ViewParams &vp) {
        const int rowsPerBand = hiresBandRows(w);
        const int bands = (hgt + rowsPerBand - 1) / rowsPerBand;
        if (ensureCapacity(spill, size_t(grid) * w * rowsPerBand) != cudaSuccess) { setError("raster spill slab allocation failed"); return MV_ERR_CUDA; }
        MvConsts k;
        fillConsts(k, w, hgt);
        vp = frameParams(w, hgt, bands, rowsPerBand, spill.p, triCap, k);
        return MV_OK;
    }
    // One camera launch on the stream: camera c of n draws env dEnv[c] (an all-zero frame outside [0, E)) through the view matrix
    // dViews[c * 16 ..] into frame c of obs / depth / seg (depth and seg may be null) at w x h, from the instance lists of the last step.
    // Stream-ordered, no ready stamps, no costs: the next step's cost-ordered queue does not see it.  The out-of-range counter is zeroed
    // first and counts this launch only.
    int launchCameras(const int32_t *dEnv, const float *dViews, int n, int w, int hgt, uint8_t *obs, float *depth, uint16_t *seg) {
        if (ensureCapacity(cams.d_range, 1) != cudaSuccess) { setError("camera counter allocation failed"); return MV_ERR_CUDA; }
        MV_CUDA(cudaMemsetAsync(cams.d_range.p, 0, sizeof(uint32_t), stream));
        if (n == 0) return MV_OK;
        mvr::ViewParams vp;
        const int rc = bandedFrame(w, hgt, cameraGrid, cams.spill, vp);
        if (rc) return rc;
        vp.instances = d_inst.p; vp.instCounts = d_instCounts.p; vp.views = dViews;
        vp.obs = obs; vp.depth = depth; vp.seg = seg;
        vp.viewBase = 0; vp.N = n;
        vp.camEnv = dEnv; vp.numEnvs = E; vp.rangeCount = cams.d_range.p;
        return launchView(vp, false, mvr::Items::Cameras);
    }
    // the host-facing camera call: tables up, draw into the engine's buffers, copy into their pinned twins, wait
    int drawCameras(const int32_t *envs, const float *views, int n, int w, int hgt, bool depth, bool seg) {
        int rc = drain();
        if (rc) return rc;
        const size_t px = size_t(n) * size_t(w) * size_t(hgt);
        const bool ok = ensureCapacity(cams.d_env, size_t(n)) == cudaSuccess && ensureCapacity(cams.d_views, size_t(n) * 16) == cudaSuccess &&
                        ensureCapacity(cams.d_obs, px * 4) == cudaSuccess && ensureCapacity(cams.h_obs, px * 4) == cudaSuccess &&
                        (!depth || (ensureCapacity(cams.d_depth, px) == cudaSuccess && ensureCapacity(cams.h_depth, px) == cudaSuccess)) &&
                        (!seg || (ensureCapacity(cams.d_seg, px) == cudaSuccess && ensureCapacity(cams.h_seg, px) == cudaSuccess)) &&
                        ensureCapacity(cams.h_range, 1) == cudaSuccess;
        if (!ok) { setError("camera buffers: allocation failed"); return MV_ERR_CUDA; }
        if (n > 0) {
            MV_CUDA(cudaMemcpyAsync(cams.d_env.p, envs, sizeof(int32_t) * size_t(n), cudaMemcpyHostToDevice, stream));
            MV_CUDA(cudaMemcpyAsync(cams.d_views.p, views, sizeof(float) * 16 * size_t(n), cudaMemcpyHostToDevice, stream));
        }
        rc = launchCameras(cams.d_env.p, cams.d_views.p, n, w, hgt, cams.d_obs.p, depth ? cams.d_depth.p : nullptr, seg ? cams.d_seg.p : nullptr);
        if (rc) return rc;
        if (n > 0) {
            MV_CUDA(cudaMemcpyAsync(cams.h_obs.p, cams.d_obs.p, px * 4, cudaMemcpyDeviceToHost, stream));
            if (depth) MV_CUDA(cudaMemcpyAsync(cams.h_depth.p, cams.d_depth.p, px * sizeof(float), cudaMemcpyDeviceToHost, stream));
            if (seg) MV_CUDA(cudaMemcpyAsync(cams.h_seg.p, cams.d_seg.p, px * sizeof(uint16_t), cudaMemcpyDeviceToHost, stream));
        }
        MV_CUDA(cudaMemcpyAsync(cams.h_range.p, cams.d_range.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        MV_CUDA(cudaStreamSynchronize(stream));
        return MV_OK;
    }
    // world-space box {min x, y, z, max x, y, z} of env e's live level from the host mirrors: static boxes (rotated ones by their extent
    // about y), decorations (a unit mesh's reach along each column, the capsule's y doubled) and terrain slabs
    void levelBounds(int e, float *out6) const {
        const size_t row = liveRow(e);
        const MvLevel &L = levels.level(row);
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        auto add = [&](const float c[3], const float r[3]) {
            for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], c[a] - r[a]); hi[a] = std::max(hi[a], c[a] + r[a]); }
        };
        const MvBox *st = levels.statics(row);
        const float *rot = levels.rotations(row);
        for (int i = 0; i < L.n_static; ++i) {
            float r[3] = {st[i].h[0], st[i].h[1], st[i].h[2]};
            if (st[i].flags & MV_ROTATED) {
                const float ax = std::fabs(rot[2 * i]), az = std::fabs(rot[2 * i + 1]);
                r[0] = ax * st[i].h[0] + az * st[i].h[2];
                r[2] = az * st[i].h[0] + ax * st[i].h[2];
            }
            add(st[i].c, r);
        }
        const MvDeco *dc = levels.deco(row);
        for (int i = 0; i < L.n_deco; ++i) {
            const float *m = dc[i].model;
            const float ys = dc[i].mesh == 1 ? 2.0f : 1.0f;
            const float c[3] = {m[12], m[13], m[14]};
            float r[3];
            for (int a = 0; a < 3; ++a) r[a] = std::fabs(m[a]) + ys * std::fabs(m[4 + a]) + std::fabs(m[8 + a]);
            add(c, r);
        }
        for (int i = 0; i < L.n_terrain; ++i) {
            const int32_t *bb = L.terrain[i].bb;
            const float c[3] = {0.5f * float(bb[0] + bb[3]), float(bb[1]) + 0.025f, 0.5f * float(bb[2] + bb[5])};
            const float r[3] = {0.5f * float(bb[3] - bb[0]), 0.025f, 0.5f * float(bb[5] - bb[2])};
            add(c, r);
        }
        for (int a = 0; a < 3; ++a) {
            out6[a] = lo[a] <= hi[a] ? lo[a] : 0.0f;
            out6[3 + a] = lo[a] <= hi[a] ? hi[a] : 0.0f;
        }
    }
    // shared-memory carve-up, occupancy and the per-CTA spill slabs for the current triangle-list capacity / band count
    int configureRaster() {
        if (stream) cudaStreamSynchronize(stream);
        rasterSmem = mvr::smemLayout(triCap).total;
        int maxOptin = 0;
        MV_CUDA(cudaDeviceGetAttribute(&maxOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        if (int(rasterSmem) > maxOptin) { setError("tri_cap needs more shared memory than an SM has"); return MV_ERR_ARG; }
        for (int v = 0; v < 4; ++v) {  // the grid fits every variant a step may launch (with and without segmentation)
            const void *fn = reinterpret_cast<const void *>(viewKernelOf(mvr::Items::All, v >= 2, v & 1));
            MV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, maxOptin));  // per function, not per engine: allow the device maximum
            int perSM = 0;
            MV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fn, mvr::kThreads, rasterSmem));
            if (perSM < 1) { setError("raster kernel does not fit on an SM with this tri_cap"); return MV_ERR_CUDA; }
            rasterCtasPerSM = v ? std::min(rasterCtasPerSM, perSM) : perSM;
        }
        rasterGrid = numSMs * rasterCtasPerSM;
        int maskedPerSM = 0;
        for (int v = 0; v < 6; ++v) {  // the masked variants (terminal frames, active envs' frames) size their own grid
            const void *fn = reinterpret_cast<const void *>(viewKernelOf(v < 2 ? mvr::Items::Ended : mvr::Items::Active, v >= 4, v & 1));
            MV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, maxOptin));
            int perSM = 0;
            MV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fn, mvr::kThreads, rasterSmem));
            maskedPerSM = v ? std::min(maskedPerSM, perSM) : perSM;
        }
        maskedGrid = numSMs * std::max(1, std::min(maskedPerSM, rasterCtasPerSM));  // shares d_spill, sized by rasterGrid
        int cameraPerSM = 0;
        for (int v = 0; v < 4; ++v) {  // the camera variants size their own grid (and spill slab) from their own occupancy
            const void *fn = reinterpret_cast<const void *>(viewKernelOf(mvr::Items::Cameras, v >= 2, v & 1));
            MV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, maxOptin));
            int perSM = 0;
            MV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fn, mvr::kThreads, rasterSmem));
            cameraPerSM = v ? std::min(cameraPerSM, perSM) : perSM;
        }
        cameraGrid = numSMs * std::max(1, std::min(cameraPerSM, rasterCtasPerSM));
        bandRows = ((H / 4 + rasterBands - 1) / rasterBands) * 4;
        if (d_spill.alloc(size_t(rasterGrid) * W * bandRows) != cudaSuccess) { setError("raster spill slab allocation failed"); return MV_ERR_CUDA; }
        hires = {};  // its spill slab is sized by the grid
        return MV_OK;
    }

    // after a step (or forced reset): move the host mirrors of finished envs to the next slot of the ring and start generating the level
    // D - 1 episodes ahead into the slot just freed
    void afterFlip(const uint8_t *flipped) {
        const int D = levelSlots;
        for (int e = 0; e < E; ++e) {
            if (!flipped || flipped[e]) {
                if (levelSet) { hostEpisode[size_t(e)] += 1; continue; }  // the kernel chose a bank row: nothing to generate, nothing to upload
                hostSlot[size_t(e)] = (hostSlot[size_t(e)] + 1) % D;
                hostEpisode[size_t(e)] += 1;
                scheduleGen(e, (hostSlot[size_t(e)] + D - 1) % D, hostEpisode[size_t(e)] + D - 1);
            }
        }
    }
    // (re)build env e's staged levels, episodes after the live one in order, from its generator's current state
    void restage(int e) {
        if (levelSet) return;  // nothing is staged: every level of the set is in the bank
        for (int i = 1; i < levelSlots; ++i) scheduleGen(e, (hostSlot[size_t(e)] + i) % levelSlots, hostEpisode[size_t(e)] + i);
    }

    // per-kernel times exist only when the raster launch runs behind the first kernel (ev[1]); when the step and raster kernels overlap
    // (the dependent launch) only their union is meaningful: {-1, whole call}
    void readKernelTimes() {
        if (cudaEventQuery(ev[2]) != cudaSuccess) return;
        lastMs[0] = -1.0f; lastMs[1] = 0.0f; lastFinalMs = 0.0f; lastRaysMs = 0.0f;
        const cudaEvent_t end = lastHadRays ? evRays : ev[2];  // the ray launches come last and are timed on their own
        switch (timedAs) {
        case Timed::Union: cudaEventElapsedTime(&lastMs[1], ev[0], end); break;
        case Timed::Split: cudaEventElapsedTime(&lastMs[0], ev[0], ev[1]); cudaEventElapsedTime(&lastMs[1], ev[1], lastHadFinal ? evFinal : end); break;
        case Timed::FirstOnly: cudaEventElapsedTime(&lastMs[0], ev[0], end); break;
        }
        if (lastHadFinal) cudaEventElapsedTime(&lastFinalMs, evFinal, end);
        if (lastHadRays) cudaEventElapsedTime(&lastRaysMs, evRays, ev[2]);
    }

    int finishStep(bool copyObs, bool wait = true) {
        MV_CUDA(cudaMemcpyAsync(h_rewards.p, d_rewards.p, sizeof(float) * N, cudaMemcpyDeviceToHost, stream));
        MV_CUDA(cudaMemcpyAsync(h_dones.p, d_dones.p, E, cudaMemcpyDeviceToHost, stream));
        MV_CUDA(cudaMemcpyAsync(h_doneReasons.p, d_doneReasons.p, E, cudaMemcpyDeviceToHost, stream));
        if (autoreset) MV_CUDA(cudaMemcpyAsync(h_awaiting.p, d_awaiting.p, E, cudaMemcpyDeviceToHost, stream));
        MV_CUDA(cudaMemcpyAsync(h_trueObj.p, d_trueObj.p, sizeof(float) * N, cudaMemcpyDeviceToHost, stream));
        if (const int rc = downloadRC(stream)) return rc;
        if (levelSet) {
            MV_CUDA(cudaMemcpyAsync(h_levelIds.p, d_levelIds.p, sizeof(int32_t) * E, cudaMemcpyDeviceToHost, stream));
            publishedCall = stepCalls - 1;  // every call so far is behind this copy
        }
        if (copyObs && !rasterToHost && sliceCount <= 1) {
            const int rc = downloadViews(0, N, stream);
            if (rc) return rc;
        }
        return wait ? waitHostStep() : MV_OK;
    }
    // the end of a host-facing call: its stream and the slice downloads drained, then its kernel times
    int waitHostStep() {
        MV_CUDA(cudaStreamSynchronize(stream));
        if (sliceCount > 1 || stateCopyPending) MV_CUDA(cudaStreamSynchronize(copyStream));
        stateCopyPending = false;
        readKernelTimes();
        return MV_OK;
    }
    // the reward table, when mv_set_reward_shaping has changed it since the last upload
    int uploadRtable() {
        if (!rtableDirty) return MV_OK;
        MV_CUDA(cudaMemcpyAsync(d_rtable.p, h_rtable.p, sizeof(float) * N * MV_R_COUNT, cudaMemcpyHostToDevice, stream));
        rtableDirty = false;
        return MV_OK;
    }

    // consume one finished asynchronous step: publish its host copies, flip mirrors, schedule level generation
    int retire(Pending &p) {
        if (!p.valid) return MV_OK;
        MV_CUDA(cudaEventSynchronize(p.ev));
        std::memcpy(h_rewards.p, p.rewards.p, sizeof(float) * N);
        std::memcpy(h_dones.p, p.dones.p, E);
        std::memcpy(h_doneReasons.p, p.reasons.p, E);
        if (autoreset) std::memcpy(h_awaiting.p, p.awaiting.p, E);
        std::memcpy(h_trueObj.p, p.trueObj.p, sizeof(float) * N);
        if (levelSet) { std::memcpy(h_levelIds.p, p.levelIds.p, sizeof(int32_t) * E); publishedCall = p.call; }
        p.valid = false;
        // with two level slots the pre-staged next level of an env is delivered three calls after its episode ended: an env that finishes
        // again sooner flipped to a stale level on the device (MV_FAULT_LEVEL_NOT_READY is latched there as well) -- refuse to go on.  Counted
        // in calls whatever option "action_repeat" is: retiring, regenerating and uploading happen once per call, so the level pipeline is
        // three calls deep (the kernel's request rule, num_frames >= 3 * repeat ticks, is the same three calls counted on the device).  With
        // four slots an env ends at most once per call, and the level replacing the end of call j is uploaded before kernel j + 3, when the
        // ends of calls j, j + 1 and j + 2 have used the three staged levels at most: there is nothing to check.  Nor with a level set,
        // whose levels never arrive.  Under autoreset 1 and 2 the staged level is taken by the flip, not the end: the rule counts flips
        if (lastAsyncDone.empty()) lastAsyncDone.assign(size_t(E), -1000);
        const uint8_t *fl = flipped();
        for (int e = 0; e < E; ++e)
            if (fl[e]) {
                if (levelSlots == 2 && !levelSet && int64_t(p.step) - lastAsyncDone[size_t(e)] < 3) asyncContractBroken = true;
                lastAsyncDone[size_t(e)] = int64_t(p.step);
            }
        afterFlip(fl);
        if (asyncContractBroken) { setError("mv_step_device: an episode lasted fewer than 3 steps -- outside the asynchronous call's contract; use mv_step"); return MV_ERR_STATE; }
        return MV_OK;
    }
    int drain() {
        for (int k = 0; k < 3; ++k) {  // oldest first
            const int rc = retire(ring[(asyncSteps + k) % 3]);
            if (rc) return rc;
        }
        return MV_OK;
    }
    // asynchronous device-resident step: returns after enqueueing.  Episode bookkeeping lags two steps, which is safe with two level slots
    // because an env cannot finish twice within four steps (doneWithTimer leaves 0.3 s = 4.5 steps, scenario.hpp:114-117); with option
    // "action_repeat" k a call runs k ticks, and DESIGN.md section 2 gives the shortest natural episodes that bound k.  Option
    // "level_slots" 4 lifts the bound (see retire).  An inactive env (dActive) cannot end, so the bound holds for a subset step as well
    int stepAsync(const int32_t *dActions, const uint8_t *dEnds, const uint8_t *dActive) {
        if (!didReset) { setError("mv_step_device before mv_reset"); return MV_ERR_STATE; }
        if (hostStepPending) { const int rcp = stepEnd(); if (rcp) return rcp; }
        if (asyncContractBroken) { setError("mv_step_device: an episode lasted fewer than 3 steps -- outside the asynchronous call's contract; use mv_step"); return MV_ERR_STATE; }
        Pending &slotP = ring[asyncSteps % 3];
        int rc = bankCall();
        if (rc) return rc;
        // levels generated since the previous call go up first (done at step k-3 -> retired at call k-1 -> uploaded ahead
        // of kernel k; that env cannot flip again before step k+1), then step k-2 is retired and its regeneration jobs
        // run on the worker pool while this call's kernels are enqueued
        rc = flushUploads();
        if (rc) return rc;
        rc = retire(ring[(asyncSteps + 1) % 3]);
        if (rc) return rc;
        rc = retire(slotP);  // only if the ring wrapped without retiring
        if (rc) return rc;
        rc = uploadRtable();
        if (rc) return rc;
        chooseDelivery(false);
        rc = launchStep(stepParams(dActions, false, &slotP, dEnds, dActive), true);  // rewards / dones / true objectives land in the ring slot straight from the kernel
        if (rc) return rc;
        MV_CUDA(cudaEventRecord(slotP.ev, stream));
        slotP.valid = true;
        slotP.step = asyncSteps;
        slotP.call = stepCalls - 1;
        ++asyncSteps;
        return MV_OK;
    }
    // mv_step_stream: the device work of stepAsync, forked from stream s onto the engine stream and joined back, with nothing a stream capture
    // refuses and nothing a graph replay would repeat stale.  The per-call scalars of a host-path step become constants of the step: a
    // memset zeroes the ready stamps and the work counter, the step kernel stamps 1 (mv_reset used it, so host-path calls stamp 2 and up),
    // and the raster launches count their work from base 0.  The memset precedes the step kernel in stream order, so it has finished
    // before the raster grid, the step kernel's programmatic dependent, can start
    int stepStream(cudaStream_t s, const int32_t *dActions, const uint8_t *dEnds, const uint8_t *dActive) {
        if (!levelSet) { setError("mv_step_stream: option level_set is off (without it every episode end needs host level generation)"); return MV_ERR_STATE; }
        if (!didReset) { setError("mv_step_stream before mv_reset"); return MV_ERR_STATE; }
        if (hostStepPending) { setError("mv_step_stream: mv_step_begin is outstanding, call mv_step_end first"); return MV_ERR_STATE; }
        if (!replacements.empty()) { setError("mv_step_stream: mv_replace_levels requests are pending (host-path steps carry them out)"); return MV_ERR_STATE; }
        if (!s) s = stream;
        if (rtableDirty) {  // only before the first stream step: in stream mode mv_set_reward_shaping uploads at once
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            MV_CUDA(cudaStreamIsCapturing(s, &cs));
            if (cs != cudaStreamCaptureStatusNone) { setError("mv_step_stream: the reward shaping changed since the last step; take one step outside the capture first"); return MV_ERR_STATE; }
            if (const int rc = uploadRtable()) return rc;
        }
        if (s != stream.h) {
            MV_CUDA(cudaEventRecord(evFork, s));
            MV_CUDA(cudaStreamWaitEvent(stream, evFork, 0));
        }
        streamMode = true;
        MV_CUDA(cudaMemsetAsync(d_ready.p, 0, sizeof(uint32_t) * (size_t(E) + 1), stream));
        counterBase = 0;
        chooseDelivery(false);
        mvk::StepParams sp = stepParams(dActions, false, nullptr, dEnds, dActive);
        sp.readyStamp = 1;
        if (const int rc = launchStep(sp, true, true)) return rc;
        if (s != stream.h) {
            MV_CUDA(cudaEventRecord(evJoin, stream));
            MV_CUDA(cudaStreamWaitEvent(s, evJoin, 0));
        }
        return MV_OK;
    }
    // Stream mode: the head of every other entry point but the pointer getters.  Graph replays run on the caller's streams, unseen by the
    // host: wait for the whole device, retire the asynchronous ring, refresh the host mirrors of what the last step left in HBM (level ids,
    // episode counters, rewards, dones, reasons, true objectives) and restart the work counter.  An outstanding mv_step_begin keeps its
    // own mirrors: mv_step_end publishes them
    int streamSync() {
        MV_CUDA(cudaDeviceSynchronize());
        MV_CUDA(cudaMemset(workCounter(), 0, sizeof(uint32_t)));
        counterBase = 0;
        if (hostStepPending) return MV_OK;
        if (const int rc = drain()) return rc;
        MV_CUDA(cudaMemcpy(h_levelIds.p, d_levelIds.p, sizeof(int32_t) * size_t(E), cudaMemcpyDeviceToHost));
        publishedCall = stepCalls - 1;
        static_assert(sizeof(MvEnvState::episode_idx) == sizeof(int), "hostEpisode mirrors MvEnvState::episode_idx");
        MV_CUDA(cudaMemcpy2D(hostEpisode.data(), sizeof(int), &d_envs.p[0].episode_idx, sizeof(MvEnvState), sizeof(int), size_t(E), cudaMemcpyDeviceToHost));
        MV_CUDA(cudaMemcpy(h_rewards.p, d_rewards.p, sizeof(float) * size_t(N), cudaMemcpyDeviceToHost));
        MV_CUDA(cudaMemcpy(h_dones.p, d_dones.p, size_t(E), cudaMemcpyDeviceToHost));
        MV_CUDA(cudaMemcpy(h_doneReasons.p, d_doneReasons.p, size_t(E), cudaMemcpyDeviceToHost));
        MV_CUDA(cudaMemcpy(h_trueObj.p, d_trueObj.p, sizeof(float) * size_t(N), cudaMemcpyDeviceToHost));
        if (autoreset) MV_CUDA(cudaMemcpy(h_awaiting.p, d_awaiting.p, size_t(E), cudaMemcpyDeviceToHost));
        noteAwaiting();  // the level set's episode counters were just read back: no flip is left to count
        return MV_OK;
    }

    int stepCommon(const int32_t *dActions, bool copyObs, bool split = false, const uint8_t *dActive = nullptr) {
        if (!didReset) { setError("mv_step before mv_reset"); return MV_ERR_STATE; }
        if (hostStepPending) { setError("mv_step_begin is outstanding: call mv_step_end first"); return MV_ERR_STATE; }
        int rc = bankCall();
        if (rc) return rc;
        rc = drain();
        if (rc) return rc;
        rc = flushUploads();
        if (rc) return rc;
        rc = uploadRtable();
        if (rc) return rc;
        chooseDelivery(copyObs);
        rc = launchStep(stepParams(dActions, false, nullptr, nullptr, dActive), true);
        if (rc) return rc;
        rc = finishStep(copyObs, !split);
        if (rc) return rc;
        if (split) { hostStepPending = true; return MV_OK; }
        afterFlip(flipped());
        return MV_OK;
    }
    // second half of a split host-facing step (mv_step_begin / mv_step_end): wait for the copies enqueued by stepCommon(split)
    int stepEnd() {
        if (!hostStepPending) { setError("mv_step_end without mv_step_begin"); return MV_ERR_STATE; }
        const int rc = waitHostStep();
        if (rc) return rc;
        hostStepPending = false;
        std::memset(h_actions.p, 0, sizeof(int32_t) * N);  // env.cpp:140-142: actions are cleared after every step
        afterFlip(flipped());
        return MV_OK;
    }
    // mv_step, and mv_step_envs with the active mask in d_active: the action masks of mv_set_actions go up, one synchronous host-facing step
    int stepHost(const uint8_t *dActive) {
        if (!didReset) { setError("mv_step before mv_reset"); return MV_ERR_STATE; }
        if (hostStepPending) { setError("mv_step_begin is outstanding: call mv_step_end first"); return MV_ERR_STATE; }
        if (cudaMemcpyAsync(d_actions.p, h_actions.p, sizeof(int32_t) * N, cudaMemcpyHostToDevice, stream) != cudaSuccess) { setError("actions upload failed"); return MV_ERR_CUDA; }
        const int rc = stepCommon(d_actions.p, obsToHost, false, dActive);
        if (rc) cudaStreamSynchronize(stream);  // the uploads may still be reading the pinned masks
        std::memset(h_actions.p, 0, sizeof(int32_t) * N);  // env.cpp:140-142: actions are cleared after every step
        return rc;
    }

    // ------------------------------------------------------------------ state stores (mv_states_*)
    // every per-env device row, in the order of StateStore::slabs, at the engine's pitches or, for growStatics, at the grown ones
    std::array<EnvSlab, kSlabCount> envSlabs() { return envSlabs(levels.staticCap, instCap()); }
    std::array<EnvSlab, kSlabCount> envSlabs(int staticPitch, int instPitch) {
        auto s = [](void *p, int units, size_t bytes) { return EnvSlab{static_cast<uint8_t *>(p), units, bytes}; };
        // with a level set a row holds no level: the bank is shared and immutable, MvEnvState names the row.  The levels' place in the
        // list is taken by the env's level id, so that a loaded env reports its level before it is stepped again
        const int D = levelSet ? 0 : levelSlots;
        const EnvSlab levelsOrId = levelSet ? s(d_levelIds.p, 1, sizeof(int32_t)) : s(levels.d_levels.p, D, sizeof(MvLevel));
        return {{s(d_envs.p, 1, sizeof(MvEnvState)), s(d_agents.p, 1, sizeof(MvAgent) * A), s(d_objects.p, 1, sizeof(MvObject) * MV_MAX_OBJECTS),
                 s(d_objGrid.p, 1, size_t(gridCells)), s(d_inst.p, 1, sizeof(MvInstance) * instPitch), s(d_instCounts.p, 1, sizeof(int32_t) * 8),
                 s(d_views.p, 1, sizeof(float) * 16 * A), levelsOrId, s(levels.d_statics.p, D, sizeof(MvBox) * staticPitch),
                 s(levels.d_staticRot.p, D, sizeof(float) * 2 * staticPitch), s(levels.d_deco.p, D, sizeof(MvDeco) * levels.decoCap),
                 s(levels.d_solid.p, D, sizeof(uint32_t) * 3 * levels.gridWords), s(d_rewards.p, 1, sizeof(float) * A), s(d_dones.p, 1, 1),
                 s(d_trueObj.p, 1, sizeof(float) * A), s(d_faults.p, 1, sizeof(int32_t)), s(d_doneReasons.p, 1, 1)}};
    }
    size_t stateRowBytes() {
        size_t b = 0;
        for (const EnvSlab &s : envSlabs()) b += s.rowBytes();
        for (int k = 0; k < 4 && wantState; ++k) b += stateRowBytes(k);
        if (wantRC) b += 3 * rcRowBytes();
        return b;
    }
    int statesCreate(int rows, int *id) {
        auto st = std::make_unique<StateStore>();
        st->rows = rows;
        const auto sl = envSlabs();
        for (int k = 0; k < kSlabCount; ++k)
            if (st->slabs[k].alloc(size_t(rows) * sl[size_t(k)].rowBytes()) != cudaSuccess) { setError("mv_states_create: allocation failed"); return MV_ERR_CUDA; }
        for (int k = 0; k < 4 && wantState; ++k)
            if (st->stateSlabs[k].alloc(size_t(rows) * stateRowBytes(k)) != cudaSuccess) { setError("mv_states_create: allocation failed"); return MV_ERR_CUDA; }
        for (int k = 0; k < 3 && wantRC; ++k)
            if (st->rcSlabs[k].alloc(size_t(rows) * rcRowBytes()) != cudaSuccess) { setError("mv_states_create: allocation failed"); return MV_ERR_CUDA; }
        st->host.resize(size_t(rows));
        stores.push_back(std::move(st));
        *id = int(stores.size()) - 1;
        return MV_OK;
    }
    // a save or load is a synchronisation point: outstanding asynchronous steps are retired and every generated level is uploaded first,
    // so that no generation job still in flight can later overwrite a restored pre-staged slot
    int quiesce() {
        const int rc = drain();
        return rc ? rc : flushUploads();
    }
    // one copy kernel over all listed rows.  toStore: engine row pairs[i].x -> store row pairs[i].y; else back, and every view is drawn
    // again behind the copy
    int copyStateRows(StateStore &st, const int32_t *from, const int32_t *to, int n, bool toStore) {
        if (size_t(n) > std::min(h_pairs.n, d_pairs.n)) {
            MV_CUDA(cudaStreamSynchronize(stream));  // the previous upload may still read the pinned pairs
            if (h_pairs.alloc(size_t(n)) != cudaSuccess || d_pairs.alloc(size_t(n)) != cudaSuccess) { setError("state pairs: allocation failed"); return MV_ERR_CUDA; }
        }
        for (int i = 0; i < n; ++i) h_pairs.p[i] = make_int2(from[i], to[i]);
        MV_CUDA(cudaMemcpyAsync(d_pairs.p, h_pairs.p, sizeof(int2) * size_t(n), cudaMemcpyHostToDevice, stream));
        const auto sl = envSlabs();
        mvs::Slab table[kSlabCount];
        for (int k = 0; k < kSlabCount; ++k) {
            uint8_t *eng = sl[size_t(k)].base, *sto = st.slabs[k].p;
            const size_t rb = sl[size_t(k)].rowBytes();
            table[k] = mvs::Slab{toStore ? eng : sto, toStore ? sto : eng, rb, rb, rb};
        }
        MV_CUDA(cudaEventRecord(ev[0], stream));
        MV_CUDA(mvs::copyRows(table, kSlabCount, d_pairs.p, n, stream));
        launches += 1;
        // the rows of the options' tensors (state tensors, reward components): a second launch of the same kernel, so that the first table
        // keeps its size
        mvs::Slab optTable[7];
        int nOpt = 0;
        auto optSlab = [&](float *engRows, uint8_t *sto, size_t rb) {
            uint8_t *eng = reinterpret_cast<uint8_t *>(engRows);
            optTable[nOpt++] = mvs::Slab{toStore ? eng : sto, toStore ? sto : eng, rb, rb, rb};
        };
        for (int k = 0; k < 4 && wantState; ++k) optSlab(stateTensor(d_state.p, k, false), st.stateSlabs[k].p, stateRowBytes(k));
        for (int k = 0; k < 3 && wantRC; ++k) optSlab(rcTensor(d_rc.p, k), st.rcSlabs[k].p, rcRowBytes());
        if (nOpt) {
            MV_CUDA(mvs::copyRows(optTable, nOpt, d_pairs.p, n, stream));
            launches += 1;
        }
        if (toStore) return endTimes(Timed::FirstOnly);
        if (const int rc = downloadState()) return rc;  // the loaded rows, while the views are drawn again
        MV_CUDA(cudaEventRecord(ev[1], stream));
        int rc = launchRaster(nullptr, 0);
        if (!rc && nRays) {  // the loaded envs' rays, behind the redraw (no terminal rays: the store keeps no terminal rows)
            MV_CUDA(cudaEventRecord(evRays, stream));
            rc = castRays(false, nullptr);
        }
        if (!rc) rc = endTimes(Timed::Split, true, false, nRays > 0);
        return (rc || !nRays) ? rc : downloadRays(stream);
    }
    // a state load or an env restart ends like a host-facing step: `launch` enqueues its kernel with every view drawn again behind it
    // (the views it did not change yield the same bytes), `whileDrawing` is the host's part, run while the device works, and frames and
    // results are delivered as a step delivers them
    template <class Launch, class Host> int redrawAndDeliver(Launch &&launch, Host &&whileDrawing) {
        chooseDelivery(obsToHost);
        int rc = launch();
        if (!rc) rc = whileDrawing();
        return rc ? rc : finishStep(obsToHost);
    }
    int statesSave(StateStore &st, const int32_t *envs, const int32_t *rows, int n) {
        int rc = quiesce();
        if (rc) return rc;
        rc = copyStateRows(st, envs, rows, n, true);
        if (rc) return rc;
        for (int i = 0; i < n; ++i) {  // host state; the workers are idle (flushUploads waited for them)
            const int e = envs[i];
            StateStore::HostRow &r = st.host[size_t(rows[i])];
            r.saved = true;
            r.scenario = envScenarioName[size_t(e)];
            r.slot = hostSlot[size_t(e)]; r.episode = hostEpisode[size_t(e)];
            if (levelSet) {  // no generator, no mirrors: the pick seed and the live row travel in MvEnvState
                r.bankRow = int(liveRow(e));
                r.bankSeed = rowSeed[size_t(r.bankRow)];
                continue;
            }
            r.gen = gens[size_t(e)];
            r.levels.clear();
            for (int s = 0; s < levelSlots; ++s) r.levels.push_back(levels.read(rowOfSlot(e, s)));
        }
        MV_CUDA(cudaStreamSynchronize(stream));
        readKernelTimes();
        return MV_OK;
    }
    // the loaded views then show the frames the saved step returned, and rewards / dones / true objectives read as they did after it
    int statesLoad(StateStore &st, const int32_t *rows, const int32_t *envs, int n) {
        const int rc = quiesce();
        if (rc) return rc;
        const int rcl = redrawAndDeliver(
            [&] {
                const int rcc = copyStateRows(st, rows, envs, n, false);
                // the loaded envs' flags (MvEnvState::pad[1], 0 or 1: its low byte) into the awaiting array, before it is delivered
                if (!rcc && autoreset) MV_CUDA(cudaMemcpy2DAsync(d_awaiting.p, 1, &d_envs.p[0].pad[1], sizeof(MvEnvState), 1, size_t(E), cudaMemcpyDeviceToDevice, stream));
                return rcc;
            },
            [&] { restoreHostRows(st, rows, envs, n); return MV_OK; });
        if (!rcl) noteAwaiting();
        return rcl;
    }
    // host state and mirrors; no episode end: no afterFlip, no generation job
    void restoreHostRows(const StateStore &st, const int32_t *rows, const int32_t *envs, int n) {
        for (int i = 0; i < n; ++i) {
            const int e = envs[i];
            const StateStore::HostRow &r = st.host[size_t(rows[i])];
            if (r.gen) gens[size_t(e)] = *r.gen;
            hostSlot[size_t(e)] = r.slot; hostEpisode[size_t(e)] = r.episode;
            for (size_t s = 0; s < r.levels.size(); ++s) levels.write(rowOfSlot(e, int(s)), r.levels[s]);  // the store's slot count is the engine's
            if (!lastAsyncDone.empty()) lastAsyncDone[size_t(e)] = -1000;  // the loaded env's last episode end is not this engine's
        }
    }

    // ------------------------------------------------------------------ per-env restart (mv_reset_envs)
    // The forced flip of mv_reset over the listed envs only (the step kernel steps sp.envOrder[0..n)), then a re-render of the batch as after
    // a state load.  A synchronisation point: on return the restarted envs' levels after next are generated and uploaded, so the
    // asynchronous call's three-step rule holds from the next mv_step_device on.
    int resetEnvs(const int32_t *envs, const int32_t *seeds, int n) {
        int rc = bankCall();
        if (rc) return rc;
        rc = quiesce();
        if (rc) return rc;
        if (seeds) {  // the staged slots take the first levels of the new stream, in order, as in a fresh engine; the workers are idle after quiesce
            for (int i = 0; i < n; ++i) {
                const int e = envs[i];
                gens[size_t(e)].restart((unsigned long)seeds[i]);
                restage(e);
                pickSeed[size_t(e)] = uint32_t(seeds[i]);  // with a level set a seed names a pick sequence, not a stream
                if ((rc = uploadPickSeeds(e, 1))) return rc;
            }
            rc = flushUploads();
            if (rc) return rc;
        }
        for (int i = 0; i < n; ++i) h_envList.p[i] = uint32_t(envs[i]);
        MV_CUDA(cudaMemcpyAsync(d_envList.p, h_envList.p, sizeof(uint32_t) * size_t(n), cudaMemcpyHostToDevice, stream));
        mvk::StepParams sp = stepParams(d_actions.p, true, nullptr, nullptr);
        sp.envOrder = d_envList.p; sp.E = n;
        rc = redrawAndDeliver([&] { return launchStep(sp, false); }, [&] {
            std::vector<uint8_t> flipped(size_t(E), 0);
            for (int i = 0; i < n; ++i) {
                flipped[size_t(envs[i])] = 1;
                if (!lastAsyncDone.empty()) lastAsyncDone[size_t(envs[i])] = -1000;  // a restart is not an asynchronous episode end
            }
            afterFlip(flipped.data());  // the levels after next, generated while the device draws
            return flushUploads();
        });
        if (!rc) noteAwaiting();  // the restart's own flips are counted above
        return rc;
    }

    // ------------------------------------------------------------------ level set
    // pickSeed[first .. first + count) into the envs' MvEnvState (after the first reset, which otherwise writes them itself), in stream
    // order behind the steps already enqueued
    int uploadPickSeeds(int first, int count) {
        if (!levelSet || !didReset) return MV_OK;
        static_assert(sizeof(MvEnvState::pad[0]) == sizeof(uint32_t), "the pick seed lives in MvEnvState::pad[0]");
        MV_CUDA(cudaMemcpy2DAsync(&d_envs.p[first].pad[0], sizeof(MvEnvState), &pickSeed[size_t(first)], sizeof(uint32_t), sizeof(uint32_t), size_t(count),
                                  cudaMemcpyHostToDevice, stream));
        MV_CUDA(cudaStreamSynchronize(stream));  // pageable source
        return MV_OK;
    }
    // option "level_set": the bank's rows replace the slot rings, and the per-env arrays of the mode appear
    int allocLevelSet() {
        if (const int rc = allocLevelSlots("level_set")) return rc;
        if (!levelSet) return MV_OK;
        const size_t n = size_t(E);
        bool ok = d_bankBase.alloc(n) == cudaSuccess && d_levelIds.alloc(n) == cudaSuccess && d_nextLevels.alloc(n) == cudaSuccess &&
                  h_levelIds.alloc(n) == cudaSuccess && h_nextLevels.alloc(n) == cudaSuccess;
        for (auto &p : ring) ok = ok && p.levelIds.alloc(n) == cudaSuccess;
        if (!ok) { setError("level_set: allocation failed"); return MV_ERR_CUDA; }
        std::memset(h_levelIds.p, 0, sizeof(int32_t) * n);
        for (auto &p : ring) std::memset(p.levelIds.p, 0, sizeof(int32_t) * n);
        std::vector<int32_t> base(n);
        for (size_t e = 0; e < n; ++e) base[e] = envBank[e] * levelSet;
        MV_CUDA(cudaMemcpy(d_bankBase.p, base.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice));
        MV_CUDA(cudaMemset(d_levelIds.p, 0, sizeof(int32_t) * n));
        MV_CUDA(cudaMemset(d_nextLevels.p, 0xFF, sizeof(int32_t) * n));  // -1: the engine picks
        rowRetiring.assign(levelRows(), 0);
        rowPickable.assign(levelRows(), 1);
        if (d_rowPickable.alloc(levelRows()) != cudaSuccess) { setError("level_set: allocation failed"); return MV_ERR_CUDA; }
        MV_CUDA(cudaMemset(d_rowPickable.p, 1, levelRows()));
        return MV_OK;
    }
    // first reset with a level set: every level of the bank, on the worker pool; flushUploads then grows the static-box arrays once, to
    // the largest level of the bank, and uploads the rows
    void scheduleBank() {
        rowSeed.resize(levelRows());
        for (int b = 0; b < numBanks; ++b)
            for (int j = 0; j < levelSet; ++j) {
                const int f = bankFirstEnv(b), row = b * levelSet + j, seed = levelSetSeed + j;
                rowSeed[size_t(row)] = seed;
                pool->submit([this, f, row, seed] { generateBankLevel(gens[size_t(f)], envScenario[size_t(f)], row, seed); });
            }
    }
    int bankFirstEnv(int b) const { return int(std::find(envBank.begin(), envBank.end(), b) - envBank.begin()); }

    // ------------------------------------------------------------------ replaceable rows (mv_replace_levels)
    // mv_replace_levels after its checks: the rows retire at the next kernel-enqueuing call; their levels are generated meanwhile
    void replaceLevels(const int32_t *rows, const int32_t *seeds, int n) {
        if (!replacePool) replacePool = std::make_unique<WorkerPool>(threads);
        for (int i = 0; i < n; ++i) {
            auto rep = std::make_unique<Replacement>();
            rep->row = rows[i]; rep->seed = seeds[i];
            rowRetiring[size_t(rows[i])] = 1;
            const int f = bankFirstEnv(rows[i] / levelSet);
            Replacement *side = rep.get();
            // the generator is copied here, on the caller's thread: mv_seed and mv_reset_envs may reseed gens[f] while the job runs
            replacePool->submit([this, gen = gens[size_t(f)], sc = envScenario[size_t(f)], side] { generateBankLevel(gen, sc, side->row, side->seed, side); });
            replacements.push_back(std::move(rep));
        }
    }
    // the start of every call that enqueues the step kernel: with a level set, the rewrites that are due, then the requests made since the
    // previous such call become retiring, and the pickable bytes go up in one copy when they changed.  Nothing at all without requests
    int bankCall() {
        const int64_t call = stepCalls++;
        if (!levelSet || replacements.empty()) return MV_OK;
        std::vector<uint8_t> held(levelRows(), 0);  // rows with an env on them as of call publishedCall
        for (int e = 0; e < E; ++e) held[size_t(envBank[size_t(e)]) * size_t(levelSet) + size_t(h_levelIds.p[e])] = 1;
        bool changed = false, staged = false;
        for (auto it = replacements.begin(); it != replacements.end();) {
            Replacement &r = **it;
            if (r.call < 0) {
                r.call = call;
                rowPickable[size_t(r.row)] = 0;
                changed = true;
            }
            if (r.call >= call || publishedCall < r.call || held[size_t(r.row)]) { ++it; continue; }
            {  // due: wait for its level if the worker has not finished it
                std::unique_lock<std::mutex> lk(genMutex);
                replaceDone.wait(lk, [&] { return r.ready; });
            }
            if (!r.error.empty()) {  // as for the bank: sticky, only mv_close recovers
                { std::lock_guard<std::mutex> lk(genMutex); genErrors.push_back(r.error); }
                setError("level generation failed: " + r.error);
                return MV_ERR_CAPACITY;
            }
            if (int(r.out.statics.size()) > levels.staticCap) {
                if (const int rc = growStatics(int(r.out.statics.size()))) return rc;
            }
            stageLevel(r.row, r.out);
            rowSeed[size_t(r.row)] = r.seed;
            rowRetiring[size_t(r.row)] = 0;
            rowPickable[size_t(r.row)] = 1;
            changed = staged = true;
            it = replacements.erase(it);
        }
        if (staged) { if (const int rc = flushUploads()) return rc; }
        // pageable source: staged before the call returns, so the vector may change at once
        if (changed) MV_CUDA(cudaMemcpyAsync(d_rowPickable.p, rowPickable.data(), rowPickable.size(), cudaMemcpyHostToDevice, stream));
        return MV_OK;
    }
    // mv_set_next_levels: the listed entries of the next-level array, in stream order ahead of the next kernel; runs of consecutive envs
    // go up in one copy
    int setNextLevels(const int32_t *envs, const int32_t *levels, int n) {
        MV_CUDA(cudaStreamSynchronize(stream));  // a previous call's copies may still read the staging array
        for (int i = 0; i < n; ++i) h_nextLevels.p[envs[i]] = levels[i];
        for (int i = 0; i < n;) {
            int len = 1;
            while (i + len < n && envs[i + len] == envs[i] + len) ++len;
            MV_CUDA(cudaMemcpyAsync(d_nextLevels.p + envs[i], h_nextLevels.p + envs[i], sizeof(int32_t) * size_t(len), cudaMemcpyHostToDevice, stream));
            i += len;
        }
        return MV_OK;
    }

    // test hook (mv_debug_warp_agent): w16 = pos[3], basis[9], hvel[3], vvel -- the head of MvAgent, written in one copy after the
    // asynchronous ring is retired.  Every other position-derived value (colliders, candidate lists, object_t, views) is rebuilt from
    // MvAgent::pos by the next step kernel.
    int warpAgent(int env, int agent, const float *w16) {
        static_assert(offsetof(MvAgent, basis) == 12 && offsetof(MvAgent, hvel) == 48 && offsetof(MvAgent, vvel) == 60, "MvAgent head layout");
        const int rc = quiesce();
        if (rc) return rc;
        MV_CUDA(cudaMemcpyAsync(&d_agents.p[size_t(env) * A + agent], w16, sizeof(float) * 16, cudaMemcpyHostToDevice, stream));
        MV_CUDA(cudaStreamSynchronize(stream));
        return MV_OK;
    }

    // Every member releases what it owns, in reverse order of declaration.  That order alone is not safe: the level workers (pool) write
    // into the pinned mirrors declared after it, replacePool's jobs into `replacements`, and both streams may still run work that reads or
    // writes the buffers.  So the workers are joined and the streams drained first.  Runs on the engine's device (mv_close, mv_create).
    ~mv_engine() {
        if (pool) { pool->waitAll(); pool.reset(); }
        replacePool.reset();  // joins its workers after the queue drains: no job outlives `replacements`
        if (stream) cudaStreamSynchronize(stream);
        if (copyStream) cudaStreamSynchronize(copyStream);
    }
};

namespace {

const uint32_t kPaletteRgb[22] = {0xffdd3c, 0x3bb372, 0x50c878, 0x2eb5d0, 0xadd8e6, 0x3a7fa6, 0x2c3e50, 0xffb400, 0xb3b3b3, 0x555555, 0x222222,
                                  0xffffff, 0xff0000, 0xffa770, 0xd468ee, 0xffe6e6, 0xffffe6, 0xccffcc, 0xe6ecff, 0xd9d9d9, 0xf2e6ff, 0xffebcc};

cudaError_t uploadPalette() {
    float pal[22][3];
    for (int i = 0; i < 22; ++i) {  // toRgbf: byte / 255 (util/magnum.hpp:25-32)
        pal[i][0] = float((kPaletteRgb[i] >> 16) & 255) / 255.0f;
        pal[i][1] = float((kPaletteRgb[i] >> 8) & 255) / 255.0f;
        pal[i][2] = float(kPaletteRgb[i] & 255) / 255.0f;
    }
    return cudaMemcpyToSymbol(mvr::c_palette, pal, sizeof(pal));
}

int setKernelAttrs(mv_engine *h) {
    cudaError_t err = cudaSuccess;
    for (int v = 0; v < 24 && err == cudaSuccess; ++v) {
        const bool rc = (v & 4) != 0;
        const int smem = int((sizeof(mvk::WarpShared) + (rc ? mvk::kRcTickBytes : 0)) * 4);
        err = cudaFuncSetAttribute(reinterpret_cast<const void *>(stepKernelOf(v & 1, v & 2, rc, v >> 3)), cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    }
    if (err != cudaSuccess) { h->setError(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(err)); return MV_ERR_CUDA; }
    return MV_OK;
}

}  // namespace

static void fillConsts(MvConsts &k, int W, int H) {
    k.dt = 1.0f / 15.0f;                              // env.hpp:160-161
    mvh::yawBasis(3.5f * k.dt, k.look_left);          // agent.cpp:100-108,128-133
    mvh::yawBasis(-3.5f * k.dt, k.look_right);
    k.max_slope_cos = mvh::crcos(45.0f * (3.14159265358979323846f / 180.0f));
    const float aspect = float(W) / float(H);
    const float halfTan = mvh::crtan((100.0f * 0.01745329251994329576923690768489f) / 2.0f);
    const float nearZ = 0.01f, farZ = 120.0f;
    k.p00 = 1.0f / halfTan;
    k.p11 = -aspect / halfTan;
    k.p22 = farZ / (nearZ - farZ);
    k.p32 = farZ * nearZ / (nearZ - farZ);
}

// In stream mode an entry point is a synchronisation point: its head is mv_engine::streamSync, and its tail waits for the work it put on
// the engine stream, which later graph replays on the caller's streams are not ordered behind.  Without stream steps both are one test
namespace {
struct StreamTail {
    mv_engine *h;
    ~StreamTail() { if (h->streamMode) cudaStreamSynchronize(h->stream); }
};
int streamHead(mv_engine *h) {
    if (!h->streamMode) return MV_OK;
    DeviceGuard dg(h->device);
    if (!dg.ok) { h->setError("cudaSetDevice failed"); return MV_ERR_CUDA; }
    return h->streamSync();
}
}  // namespace
#define MV_SYNC_POINT(h)                                                                                          \
    StreamTail tail__{(h)};                                                                                       \
    if (const int rcs__ = streamHead(h)) return rcs__;
// the calls that would reallocate or re-pitch a buffer a captured launch refers to
#define MV_NOT_IN_STREAM_MODE(h, what)                                                                            \
    if ((h)->streamMode) { (h)->setError(std::string(what) + ": refused after mv_step_stream (a captured launch may refer to the buffers it reallocates)"); return MV_ERR_STATE; }

extern "C" {

const char *mv_last_error(mv_handle h) { return h ? h->error.c_str() : g_createError.c_str(); }

int mv_create(const char *scenario, int w, int h, int num_envs, int num_agents, int num_threads, int device, const char *const *keys, const float *vals,
              int nparams, mv_handle *out) {
    const std::vector<const char *> names(size_t(std::max(num_envs, 0)), scenario);
    return mv_create_mixed(names.data(), w, h, num_envs, num_agents, num_threads, device, keys, vals, nparams, out);
}

int mv_create_mixed(const char *const *scenarios, int w, int h, int num_envs, int num_agents, int num_threads, int device, const char *const *keys,
                    const float *vals, int nparams, mv_handle *out) {
    if (!out) return MV_ERR_ARG;
    *out = nullptr;
    if (num_envs <= 0 || num_agents <= 0 || num_agents > MV_MAX_AGENTS) { g_createError = "bad num_envs / num_agents_per_env"; return MV_ERR_ARG; }
    if (!scenarios) { g_createError = "null scenario list"; return MV_ERR_ARG; }
    std::vector<std::string> names(static_cast<size_t>(num_envs));
    std::vector<int> scs(static_cast<size_t>(num_envs));
    for (int i = 0; i < num_envs; ++i) {
        const char *s = scenarios[i];
        scs[size_t(i)] = s ? mv::scenarioFromName(s) : -1;
        if (scs[size_t(i)] < 0) { g_createError = std::string("unknown scenario ") + (s ? s : "(null)") + " for env " + std::to_string(i); return MV_ERR_ARG; }
        names[size_t(i)] = s;
        for (char &c : names[size_t(i)]) c = char(std::tolower(static_cast<unsigned char>(c)));  // one spelling per scenario (the state store compares them)
    }
    if (w <= 0 || h <= 0 || w % 32 != 0 || h % 4 != 0 || (w / 32) * (h / 4) > 128 || w > kMaxRasterWidth) {
        g_createError = "render size must be a multiple of 32x4 with at most 128 tiles, at most 768 wide";
        return MV_ERR_ARG;
    }
    for (int i = 0; i < nparams; ++i) {
        if (!keys || !keys[i] || !vals) { g_createError = "null parameter key / value array"; return MV_ERR_ARG; }
        // the interactive viewer's reward-indicator HUD (scenario_default.hpp:144-160, set by viewer_app.cpp:147 only) adds drawables this
        // engine does not draw: refuse instead of rendering frames that differ from the reference's
        if (std::string(keys[i]) == "useUIRewardIndicators" && vals[i] > 0.0f) {
            g_createError = "useUIRewardIndicators > 0 (the viewer's reward-indicator HUD) is not supported";
            return MV_ERR_ARG;
        }
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { g_createError = "no CUDA device: megaverse_b200 has no CPU fallback"; return MV_ERR_CUDA; }
    if (device < 0 || device >= ndev) { g_createError = "bad CUDA device ordinal"; return MV_ERR_ARG; }
    auto *e = new mv_engine;
    auto fail = [&](int code) { g_createError = e->error; delete e; return code; };
    DeviceGuard dg__(device);
    if (!dg__.ok) { e->setError("cudaSetDevice failed"); return fail(MV_ERR_CUDA); }
    e->W = w; e->H = h; e->E = num_envs; e->A = num_agents; e->N = num_envs * num_agents; e->device = device;
    e->threads = num_threads < 1 ? 1 : num_threads;
    e->envScenarioName = names;
    e->envScenario = scs;
    e->shaping.resize(size_t(e->N));
    try {
        // every env starts from its own scenario's defaults and then takes the overrides (make_env_multitask passes one dict to every task)
        std::map<std::string, mv::FloatParams> params;
        std::map<std::string, std::vector<std::pair<std::string, float>>> shaping;
        for (int i = 0; i < e->E; ++i) {
            const std::string &name = names[size_t(i)];
            if (!params.count(name)) {
                mv::FloatParams &p = params[name];
                p = mv::defaultFloatParams(name);
                for (int k = 0; k < nparams; ++k) p[keys[k]] = vals[k];
                std::map<std::string, float> m{{"teamSpirit", 0.0f}};
                for (auto &kv : mv::defaultRewardShaping(name)) m[kv.first] = kv.second;
                shaping[name].assign(m.begin(), m.end());
            }
            e->gens.emplace_back(name, e->A, params[name]);
            for (int a = 0; a < e->A; ++a) e->shaping[size_t(i) * e->A + a] = shaping[name];
        }
    } catch (const std::exception &ex) {  // e.g. Sokoban without a Boxoban dataset (the reference exit()s here, scenario_sokoban.cpp:76-78)
        e->setError(ex.what());
        return fail(MV_ERR_ARG);
    }
    {   // the distinct scenario names, in order of first appearance: a level set keeps one run of bank rows for each
        std::vector<std::string> distinct;
        for (const std::string &name : names) {
            const size_t b = size_t(std::find(distinct.begin(), distinct.end(), name) - distinct.begin());
            if (b == distinct.size()) distinct.push_back(name);
            e->envBank.push_back(int(b));
        }
        e->numBanks = int(distinct.size());
        for (int i = 0; i < e->E; ++i) e->pickSeed.push_back(uint32_t(std::uniform_int_distribution<>{0, (1 << 30) - 1}(e->master)));
    }
    e->genQueue.resize(size_t(e->E));
    e->genBusy.assign(size_t(e->E), 0);
    e->pool.reset(new WorkerPool(e->threads));
    // one pitch for all envs: the largest capacity among the engine's scenarios
    for (int sc : scs) { e->gridCells = std::max(e->gridCells, mv::gridCapacity(sc)); e->levels.decoCap = std::max(e->levels.decoCap, mv::decoCapacity(sc)); }
    e->levels.gridWords = e->gridCells / 32;
    fillConsts(e->consts, w, h);

    auto ck = [&](cudaError_t err, const char *what) { if (err != cudaSuccess) { e->setError(std::string(what) + ": " + cudaGetErrorString(err)); return false; } return true; };
    const size_t E = size_t(e->E), N = size_t(e->N), px = size_t(w) * h;
    bool ok = ck(e->stream.create(cudaStreamNonBlocking), "stream") && ck(e->copyStream.create(cudaStreamNonBlocking), "copy stream");
    for (auto &evx : e->ev) ok = ok && ck(evx.create(cudaEventDefault), "event");
    ok = ok && ck(e->evFinal.create(cudaEventDefault), "event");
    ok = ok && e->allocLevelSlots("level slots") == MV_OK && ck(e->d_objGrid.alloc(E * e->gridCells), "objGrid") &&
         ck(e->d_envs.alloc(E), "envs") && ck(e->d_agents.alloc(N), "agents") && ck(e->d_objects.alloc(E * MV_MAX_OBJECTS), "objects") &&
         ck(e->d_instCounts.alloc(E * 8), "instCounts") && ck(e->d_views.alloc(N * 16), "views") &&
         ck(e->d_actions.alloc(N), "actions") && ck(e->d_rtable.alloc(N * MV_R_COUNT), "rtable") && ck(e->d_rewards.alloc(N), "rewards") &&
         ck(e->d_dones.alloc(E), "dones") && ck(e->d_doneReasons.alloc(E), "doneReasons") && ck(cudaMemset(e->d_doneReasons.p, 0, E), "doneReasons") &&
         ck(e->d_trueObj.alloc(N), "trueObj") && ck(e->d_obs.alloc(N * px * 4), "obs") && ck(e->d_faults.alloc(E), "faults") &&
         ck(e->d_viewCost.alloc(e->costItems() + size_t(E) + 1), "viewCost") && ck(e->resetViewOrder(), "viewOrder") && ck(e->d_ready.alloc(E + 1), "ready") &&
         ck(cudaMemset(e->d_ready.p, 0, sizeof(uint32_t) * (E + 1)), "ready");
    ok = ok && ck(e->evFork.create(cudaEventDisableTiming), "event") && ck(e->evJoin.create(cudaEventDisableTiming), "event");
    { cudaDeviceProp prop; if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) e->numSMs = prop.multiProcessorCount; }
    if (e->instCap() > mvr::kMaxInstancesPerEnv) { e->setError("instance capacity exceeds the draw-order key range"); return fail(MV_ERR_CAPACITY); }
    // few views: split every view into row bands so that the persistent grid (2 CTAs per SM) has something to balance; every band repeats
    // the view's geometry.  Measured on an H100 (ms per step, 1 / 2 / 3 bands): TowerBuilding 64 views 0.106 / 0.091 / 0.085, 256 views
    // 0.135 / 0.148 / 0.139, 512 views 0.185 / 0.185; Collect 256 views 0.546 / 0.425 / 0.387, 512 views 0.564 / 0.421
    e->rasterBands = N <= 320 ? 3 : (N <= 640 ? 2 : 1);
    while (e->rasterBands > 1 && (h / 4) % e->rasterBands) --e->rasterBands;
    if (ok && e->configureRaster() != MV_OK) return fail(MV_ERR_CUDA);
    ok = ok && ck(e->h_actions.alloc(N), "h_actions") &&
         ck(e->h_rtable.alloc(N * MV_R_COUNT), "h_rtable") && ck(e->h_rewards.alloc(N), "h_rewards") && ck(e->h_dones.alloc(E), "h_dones") && ck(e->h_doneReasons.alloc(E), "h_doneReasons") &&
         ck(e->h_trueObj.alloc(N), "h_trueObj") && ck(e->h_obs.alloc(N * px * 4), "h_obs") && ck(e->h_faults.alloc(E), "h_faults") && ck(e->h_faultWord.alloc(1), "h_faultWord") &&
         ck(e->h_envList.alloc(E), "h_envList") && ck(e->d_envList.alloc(E), "envList") && ck(e->h_active.alloc(E), "h_active") && ck(e->d_active.alloc(E), "active");
    for (auto &p : e->ring) ok = ok && ck(p.ev.create(cudaEventDisableTiming), "event") && ck(p.rewards.alloc(N), "ring") && ck(p.trueObj.alloc(N), "ring") && ck(p.dones.alloc(E), "ring") && ck(p.reasons.alloc(E), "ring");
    if (!ok) return fail(MV_ERR_CUDA);
    std::memset(e->h_actions.p, 0, sizeof(int32_t) * N);
    e->h_faultWord.p[0] = 0;
    std::memset(e->h_rewards.p, 0, sizeof(float) * N);
    std::memset(e->h_dones.p, 0, E);
    std::memset(e->h_doneReasons.p, 0, E);
    std::memset(e->h_trueObj.p, 0, sizeof(float) * N);
    std::memset(e->h_obs.p, 0, N * px * 4);
    for (size_t v = 0; v < N; ++v) e->fillRtableRow(int(v));
    ok = ck(cudaMemset(e->d_trueObj.p, 0, sizeof(float) * N), "memset") && ck(cudaMemset(e->d_faults.p, 0, sizeof(int32_t) * E), "memset") &&
         ck(cudaMemset(e->d_actions.p, 0, sizeof(int32_t) * N), "memset") && ck(cudaMemset(e->d_agents.p, 0, sizeof(MvAgent) * N), "memset") &&
         ck(cudaMemset(e->d_objects.p, 0, sizeof(MvObject) * E * MV_MAX_OBJECTS), "memset");
    if (!ok) return fail(MV_ERR_CUDA);
    e->obsOut = e->d_obs.p;
    if (!ck(uploadPalette(), "palette upload")) return fail(MV_ERR_CUDA);
    if (setKernelAttrs(e) != MV_OK) return fail(MV_ERR_CUDA);
    *out = e;
    return MV_OK;
}

int mv_set_option(mv_handle h, const char *key, int value) {
    if (!key) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const std::string k = key;
    if (k == "depth") {
        if (h->didReset) { h->setError("option depth must be set before the first reset"); return MV_ERR_STATE; }
        // on only once both buffers exist: a failed allocation leaves the option off and no buffer held
        if (value != 0 && !h->d_depth.p) {
            const size_t cnt = size_t(h->N) * h->W * h->H;
            if (h->d_depth.alloc(cnt) != cudaSuccess || h->h_depth.alloc(cnt) != cudaSuccess) { h->d_depth.free(); h->setError("depth allocation failed"); return MV_ERR_CUDA; }
            if (!h->depthOut) h->depthOut = h->d_depth.p;
        }
        h->wantDepth = value != 0;
        return MV_OK;
    }
    if (k == "segmentation") {  // the drawable behind every pixel (see the header); the buffers are allocated here, only when it is on
        if (h->didReset) { h->setError("option segmentation must be set before the first reset"); return MV_ERR_STATE; }
        if (value != 0 && value != 1) { h->setError("segmentation must be 0 or 1"); return MV_ERR_ARG; }
        if (value && !h->d_seg.p) {  // as for depth
            const size_t cnt = size_t(h->N) * h->W * h->H;
            if (h->d_seg.alloc(cnt) != cudaSuccess || h->h_seg.alloc(cnt) != cudaSuccess) { h->d_seg.free(); h->setError("segmentation allocation failed"); return MV_ERR_CUDA; }
        }
        h->wantSeg = value != 0;
        return MV_OK;
    }
    if (k == "final_obs") {  // terminal frames of ended episodes; the buffers are allocated by the first reset (after "depth" / "static_cap")
        if (h->didReset) { h->setError("option final_obs must be set before the first reset"); return MV_ERR_STATE; }
        if (value != 0 && h->autoreset) { h->setError("option final_obs needs option autoreset 0: under the other modes the observation is the terminal frame"); return MV_ERR_ARG; }
        h->wantFinal = value != 0;
        return MV_OK;
    }
    if (k == "autoreset") {  // what an episode end does (see the header); the flag arrays are allocated here, only under modes 1 and 2
        if (h->didReset) { h->setError("option autoreset must be set before the first reset"); return MV_ERR_STATE; }
        if (value < 0 || value > 2) { h->setError("autoreset must be 0 (same-step), 1 (next-step) or 2 (disabled)"); return MV_ERR_ARG; }
        if (value != 0 && h->wantFinal) { h->setError("option autoreset " + std::to_string(value) + " needs option final_obs 0: the observation is the terminal frame"); return MV_ERR_ARG; }
        if (value != 0 && !h->d_awaiting.p) {
            const size_t E = size_t(h->E);
            bool ok = h->d_awaiting.alloc(E) == cudaSuccess && cudaMemset(h->d_awaiting.p, 0, E) == cudaSuccess && h->h_awaiting.alloc(E) == cudaSuccess;
            for (auto &p : h->ring) ok = ok && p.awaiting.alloc(E) == cudaSuccess;
            if (!ok) { h->d_awaiting.free(); h->setError("autoreset: allocation failed"); return MV_ERR_CUDA; }
            std::memset(h->h_awaiting.p, 0, E);
            for (auto &p : h->ring) std::memset(p.awaiting.p, 0, E);
            h->awaitPrev.assign(E, 0);
            h->flips.assign(E, 0);
        }
        h->autoreset = value;
        return MV_OK;
    }
    if (k == "state_tensors") {  // agent / env / object / reward rows beside the frames (see the header); allocated by the first reset
        if (h->didReset) { h->setError("option state_tensors must be set before the first reset"); return MV_ERR_STATE; }
        if (value != 0 && value != 1) { h->setError("state_tensors must be 0 or 1"); return MV_ERR_ARG; }
        h->wantState = value != 0;
        return MV_OK;
    }
    if (k == "reward_components") {  // the reward split by shaping slot, per call and per finished episode (see the header); allocated by the first reset
        if (h->didReset) { h->setError("option reward_components must be set before the first reset"); return MV_ERR_STATE; }
        if (value != 0 && value != 1) { h->setError("reward_components must be 0 or 1"); return MV_ERR_ARG; }
        h->wantRC = value != 0;
        return MV_OK;
    }
    if (k == "action_repeat") {  // physics ticks per step call (see the header); the state store keeps no copy: it belongs to the engine
        if (h->didReset) { h->setError("option action_repeat must be set before the first reset"); return MV_ERR_STATE; }
        if (value < 1 || value > 4) { h->setError("action_repeat out of range [1,4]"); return MV_ERR_ARG; }
        h->actionRepeat = value;
        return MV_OK;
    }
    if (k == "level_slots") {  // level slots per env (see the header): every [E][D] array is allocated again, on the device and pinned
        if (h->didReset) { h->setError("option level_slots must be set before the first reset"); return MV_ERR_STATE; }
        if (value != 2 && value != 4) { h->setError("level_slots must be 2 or 4"); return MV_ERR_ARG; }
        h->levelSlots = value;
        return h->allocLevelSlots("level_slots");
    }
    if (k == "level_set" || k == "level_set_seed") {  // a fixed bank of levels instead of the endless streams (see the header)
        if (h->didReset) { h->setError("option " + k + " must be set before the first reset"); return MV_ERR_STATE; }
        if (k == "level_set_seed") { h->levelSetSeed = value; return MV_OK; }
        if (value < 0 || value > (1 << 20)) { h->setError("level_set out of range [0, 1048576]"); return MV_ERR_ARG; }
        h->levelSet = value;
        return h->allocLevelSet();
    }
    if (k == "tri_cap") {  // triangles a raster CTA keeps in shared memory; views with more are drawn in several batches
        MV_NOT_IN_STREAM_MODE(h, "option tri_cap")
        if (value < 32 || value > mvr::kMaxTriCap) { h->setError("tri_cap out of range [32,1022]"); return MV_ERR_ARG; }
        const int old = h->triCap;
        h->triCap = value;
        const int rc = h->configureRaster();
        if (rc) { h->triCap = old; h->configureRaster(); }
        return rc;
    }
    if (k == "static_cap") {  // initial size of the per-level static-box arrays (they grow on demand; tests start small to exercise that)
        if (h->didReset) { h->setError("option static_cap must be set before the first reset"); return MV_ERR_STATE; }
        if (value < 1 || value > (1 << 20)) return MV_ERR_ARG;
        h->levels.staticCap = value;
        return h->allocLevelSlots("static_cap");
    }
    if (k == "raster_bands") {  // row bands per view (each band is one work item of the persistent raster grid)
        MV_NOT_IN_STREAM_MODE(h, "option raster_bands")
        if (value < 1 || value > h->H / 4 || (h->H / 4) % value) { h->setError("raster_bands must divide the number of 4-pixel tile rows"); return MV_ERR_ARG; }
        h->rasterBands = value;
        return h->configureRaster();
    }
    if (k == "raster_sched") {  // work order of the persistent raster grid: 0 natural, 1 cost-ordered for launches with several views per CTA, 2 always
        if (value < 0 || value > 2) return MV_ERR_ARG;
        cudaStreamSynchronize(h->stream);
        h->rasterSched = value;
        return h->resetViewOrder() == cudaSuccess ? MV_OK : MV_ERR_CUDA;
    }
    if (k == "raster_grid") {  // CTAs of the persistent raster grid (0 = as many as the GPU holds): engines that share a GPU take a share each
        if (value < 0) return MV_ERR_ARG;
        cudaStreamSynchronize(h->stream);
        h->rasterGridCap = value;
        return MV_OK;
    }
    if (k == "obs_to_host") { h->obsToHost = value != 0; return MV_OK; }
    if (k == "zero_copy") { h->zeroCopyOpt = value != 0; return MV_OK; }
    if (k == "host_slices") { if (value < 0 || value > 64) return MV_ERR_ARG; h->hostSlicesOpt = value; return MV_OK; }
    if (k == "skip_unfit_levels") { h->skipUnfitLevels = value != 0; return MV_OK; }
    if (k == "fast_shading") { h->fastShading = value != 0; return MV_OK; }
    if (k == "overlap") { cudaStreamSynchronize(h->stream); h->overlap = value != 0; return MV_OK; }
    h->setError("unknown option " + k);
    return MV_ERR_ARG;
}

static void regenerateNext(mv_handle h) {
    // (re)build every env's pre-staged levels from its current RNG state
    for (int e = 0; e < h->E; ++e) h->restage(e);
}

static void ensureMirrors(mv_handle h) {
    if (h->hostSlot.empty()) {
        h->hostSlot.assign(size_t(h->E), h->levelSlots - 1);  // first flip lands on slot 0
        h->hostEpisode.assign(size_t(h->E), -1);  // ... as episode 0
    }
}

int mv_seed(mv_handle h, int seed) {
    if (!h) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    h->pool->waitAll();
    h->master.seed((unsigned long)seed);
    for (int e = 0; e < h->E; ++e) {  // one draw per env: its generator's seed, and its pick seed in a level set
        const int s = std::uniform_int_distribution<>{0, (1 << 30) - 1}(h->master);
        h->gens[size_t(e)].seed((unsigned long)s);
        h->pickSeed[size_t(e)] = uint32_t(s);
    }
    if (h->levelSet && h->didReset) {  // the bank stays; the envs' pick seeds change
        MV_ON_DEVICE(h)
        return h->uploadPickSeeds(0, h->E);
    }
    if (h->didReset) {  // the staged next levels were drawn from the old streams: redo them
        { std::lock_guard<std::mutex> lk(h->genMutex); h->pendingUpload.clear(); }
        regenerateNext(h);
    }
    return MV_OK;
}

int mv_seed_env(mv_handle h, int env, int seed) {
    if (!h || env < 0 || env >= h->E) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    h->pool->waitAll();
    h->gens[size_t(env)].seed((unsigned long)seed);
    h->pickSeed[size_t(env)] = uint32_t(seed);
    if (h->levelSet && h->didReset) {
        MV_ON_DEVICE(h)
        if (const int rc = h->uploadPickSeeds(env, 1)) return rc;
    }
    if (h->didReset) h->restage(env);  // every staged level, from the new stream in order
    return MV_OK;
}

int mv_reset(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    ensureMirrors(h);
    if (h->hostStepPending) { const int rcp = h->stepEnd(); if (rcp) return rcp; }
    if (const int rcb = h->bankCall()) return rcb;
    if (h->didReset) { const int rcd = h->drain(); if (rcd) return rcd; }
    if (!h->didReset) {
        // initial device state: the last slot / episode -1 so that the forced flip lands on (slot 0, episode 0); the first levels go to
        // slots 0 .. D - 2 as episodes 0 .. D - 2
        std::vector<MvEnvState> init(size_t(h->E));
        std::memset(init.data(), 0, sizeof(MvEnvState) * init.size());
        for (auto &s : init) { s.slot = h->levelSlots - 1; s.episode_idx = -1; mvBzInit(s); }
        // level set: any row of the bank to start from, and the pick seed with which the forced flip chooses episode 0's row
        for (int e = 0; e < h->E && h->levelSet; ++e) { init[size_t(e)].slot = 0; init[size_t(e)].pad[0] = int32_t(h->pickSeed[size_t(e)]); }
        if (cudaMemcpy(h->d_envs.p, init.data(), sizeof(MvEnvState) * init.size(), cudaMemcpyHostToDevice) != cudaSuccess) { h->setError("env init upload failed"); return MV_ERR_CUDA; }
        if (h->wantFinal) {
            const size_t E = size_t(h->E), N = size_t(h->N), px = size_t(h->W) * h->H;
            if (h->d_termInst.alloc(E * size_t(h->instCap())) != cudaSuccess || h->d_termCounts.alloc(E * 8) != cudaSuccess || h->d_termViews.alloc(N * 16) != cudaSuccess ||
                h->d_finalObs.alloc(N * px * 4) != cudaSuccess || h->h_finalObs.alloc(N * px * 4) != cudaSuccess ||
                (h->wantDepth && (h->d_finalDepth.alloc(N * px) != cudaSuccess || h->h_finalDepth.alloc(N * px) != cudaSuccess)) ||
                cudaMemset(h->d_finalObs.p, 0, N * px * 4) != cudaSuccess || (h->wantDepth && cudaMemset(h->d_finalDepth.p, 0, sizeof(float) * N * px) != cudaSuccess)) {
                h->setError("final_obs: allocation failed");
                return MV_ERR_CUDA;
            }
            std::memset(h->h_finalObs.p, 0, N * px * 4);
            if (h->wantDepth) std::memset(h->h_finalDepth.p, 0, sizeof(float) * N * px);
        }
        if (h->wantState) {  // the live rows and, with final_obs, the terminal rows: one block, zero until written
            const size_t n = h->stateBlockFloats();
            if (h->d_state.alloc(n) != cudaSuccess || h->h_state.alloc(n) != cudaSuccess || cudaMemset(h->d_state.p, 0, sizeof(float) * n) != cudaSuccess ||
                h->evState.create(cudaEventDisableTiming) != cudaSuccess) {
                h->setError("state_tensors: allocation failed");
                return MV_ERR_CUDA;
            }
            std::memset(h->h_state.p, 0, sizeof(float) * n);
        }
        if (h->wantRC) {  // step rows, episode rows, running totals: zero until written
            const size_t n = h->rcFloats();
            if (h->d_rc.alloc(3 * n) != cudaSuccess || h->h_rc.alloc(2 * n) != cudaSuccess || cudaMemset(h->d_rc.p, 0, sizeof(float) * 3 * n) != cudaSuccess) {
                h->setError("reward_components: allocation failed");
                return MV_ERR_CUDA;
            }
            std::memset(h->h_rc.p, 0, sizeof(float) * 2 * n);
        }
        if (h->nRays) {  // the fan, and the live and terminal rays: zero until cast
            const size_t n = h->rayBlock();
            if (h->d_rayDirs.alloc(size_t(h->nRays) * 3) != cudaSuccess || h->d_rayDist.alloc(n) != cudaSuccess || h->d_rayTag.alloc(n) != cudaSuccess ||
                h->h_rayDist.alloc(n) != cudaSuccess || h->h_rayTag.alloc(n) != cudaSuccess ||
                cudaMemcpy(h->d_rayDirs.p, h->rayDirs.data(), sizeof(float) * h->rayDirs.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemset(h->d_rayDist.p, 0, sizeof(float) * n) != cudaSuccess || cudaMemset(h->d_rayTag.p, 0, sizeof(uint16_t) * n) != cudaSuccess ||
                h->evRays.create(cudaEventDefault) != cudaSuccess) {
                h->setError("rays: allocation failed");
                return MV_ERR_CUDA;
            }
            std::memset(h->h_rayDist.p, 0, sizeof(float) * n);
            std::memset(h->h_rayTag.p, 0, sizeof(uint16_t) * n);
        }
        if (h->levelSet) h->scheduleBank();
        else regenerateNext(h);
        h->didReset = true;
    }
    int rc = h->flushUploads();
    if (rc) return rc;
    rc = h->uploadRtable();
    if (rc) return rc;
    h->chooseDelivery(h->obsToHost);
    rc = h->launchStep(h->stepParams(h->d_actions.p, true, nullptr, nullptr), true);
    if (rc) return rc;
    rc = h->finishStep(h->obsToHost);
    if (rc) return rc;
    h->afterFlip(nullptr);
    h->noteAwaiting();
    return MV_OK;
}

int32_t mv_encode_action(const int32_t *heads6) {  // megaverse.cpp:100-116 with Env::actionSpaceSizes {3,3,3,2,2,3}
    static const int sizes[6] = {3, 3, 3, 2, 2, 3};
    int idx = 0, mask = 0;
    for (int i = 0; i < 6; ++i) {
        if (heads6[i] > 0) mask |= 1 << (idx + heads6[i]);
        idx += sizes[i] - 1;
    }
    return mask;
}

int mv_set_actions(mv_handle h, const int32_t *masks) {
    if (!h || !masks) return MV_ERR_ARG;
    std::memcpy(h->h_actions.p, masks, sizeof(int32_t) * h->N);
    return MV_OK;
}

int mv_step(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    return h->stepHost(nullptr);
}

int mv_step_begin(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    if (cudaMemcpyAsync(h->d_actions.p, h->h_actions.p, sizeof(int32_t) * h->N, cudaMemcpyHostToDevice, h->stream) != cudaSuccess) { h->setError("actions upload failed"); return MV_ERR_CUDA; }
    return h->stepCommon(h->d_actions.p, h->obsToHost, true);
}

int mv_step_end(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    return h->stepEnd();
}

int mv_step_device(mv_handle h, const int32_t *d_masks) { return mv_step_device_ends(h, d_masks, nullptr); }

int mv_step_device_ends(mv_handle h, const int32_t *d_masks, const uint8_t *d_ends) { return mv_step_device_active(h, d_masks, d_ends, nullptr); }

int mv_step_device_active(mv_handle h, const int32_t *d_masks, const uint8_t *d_ends, const uint8_t *d_active) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    return h->stepAsync(d_masks ? d_masks : h->d_actions.p, d_ends, d_active);
}

int mv_step_stream(mv_handle h, void *stream, const int32_t *d_masks, const uint8_t *d_ends, const uint8_t *d_active) {
    MV_ON_DEVICE(h)
    return h->stepStream(static_cast<cudaStream_t>(stream), d_masks ? d_masks : h->d_actions.p, d_ends, d_active);
}

// host-only: the colour tables of the level generators followed by the rasteriser's palette (float bit patterns), in the layout of
// the oracle's / reference shim's *_color_tables
int mv_debug_color_tables(uint32_t *out, int cap) {
    std::vector<uint32_t> o = mv::colorTables();
    for (int i = 0; i < 22; ++i)
        for (float f : {float((kPaletteRgb[i] >> 16) & 255) / 255.0f, float((kPaletteRgb[i] >> 8) & 255) / 255.0f, float(kPaletteRgb[i] & 255) / 255.0f}) {
            uint32_t u; std::memcpy(&u, &f, 4); o.push_back(u);
        }
    if (int(o.size()) > cap) return -int(o.size());
    std::copy(o.begin(), o.end(), out);
    return int(o.size());
}

// host-only: a scenario's default reward shaping (as mv_create builds it) and default float parameters, as text
// "R key=bits\n" / "P key=bits\n" lines in key order, float values as 8 hex digits
int mv_debug_defaults(const char *scenario, char *out, int cap) {
    if (!scenario || mv::scenarioFromName(scenario) < 0) return MV_ERR_ARG;
    std::map<std::string, float> m{{"teamSpirit", 0.0f}};
    for (auto &kv : mv::defaultRewardShaping(scenario)) m[kv.first] = kv.second;
    std::string text;
    char line[160];
    auto put = [&](char tag, const std::string &k, float v) {
        uint32_t u; std::memcpy(&u, &v, 4);
        std::snprintf(line, sizeof(line), "%c %s=%08x\n", tag, k.c_str(), u);
        text += line;
    };
    for (auto &kv : m) put('R', kv.first, kv.second);
    for (auto &kv : mv::defaultFloatParams(scenario)) put('P', kv.first, kv.second);
    if (int(text.size()) + 1 > cap) return -int(text.size()) - 1;
    std::memcpy(out, text.c_str(), text.size() + 1);
    return int(text.size());
}

// host-only: how many levels of the env stream (seed env_seed) up to and including `episode` generateFitting had to skip, or < 0
int mv_debug_count_unfit_levels(const char *scenario, int num_agents, int env_seed, int episodes, const char *const *keys, const float *vals, int nparams) {
    if (!scenario || mv::scenarioFromName(scenario) < 0 || num_agents < 1 || num_agents > MV_MAX_AGENTS) return MV_ERR_ARG;
    try {
        mv::FloatParams params = mv::defaultFloatParams(scenario);
        for (int i = 0; i < nparams; ++i) params[keys[i]] = vals[i];
        mv::LevelGenerator gen(scenario, num_agents, params);
        gen.seed((unsigned long)env_seed);
        mv::LevelOut lo;
        int skipped = 0;
        for (int ep = 0; ep < episodes; ++ep) skipped += gen.generateFitting(lo, ep, 1 << 30);
        return skipped;
    } catch (const std::exception &ex) { g_createError = ex.what(); return MV_ERR_CAPACITY; }
}

int mv_levels_skipped(mv_handle h) { return h ? h->levelsSkipped.load() : MV_ERR_ARG; }

int mv_draw_hires(mv_handle h, int w, int hgt, const uint8_t **out) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const int rc = h->drawHires(w, hgt);
    if (rc) return rc;
    if (out) *out = h->hires.h_obs.p;
    return MV_OK;
}

// ------------------------------------------------------------------------------------------------ spectator cameras
// the checks both camera calls share: state first (nothing may change on a refused call), then the arguments
static int cameraCall(mv_handle h, const void *envs, const void *views, int n, int w, int hgt, const char *fn) {
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    if (h->hostStepPending) { h->setError(std::string(fn) + ": mv_step_begin is outstanding, call mv_step_end first"); return MV_ERR_STATE; }
    if (n < 0 || (n > 0 && (!envs || !views))) { h->setError(std::string(fn) + ": bad env / view tables"); return MV_ERR_ARG; }
    if (!hiresSizeOk(w, hgt)) { h->setError(std::string(fn) + ": camera frames must be a multiple of 32 x 4, at most 768 x 4096"); return MV_ERR_ARG; }
    return MV_OK;
}

int mv_draw_cameras(mv_handle h, const int32_t *envs, const float *views16, int n, int w, int hgt, int want_depth, int want_seg, const uint8_t **obs,
                    const float **depth, const uint16_t **seg, uint32_t *out_of_range) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = cameraCall(h, envs, views16, n, w, hgt, "mv_draw_cameras");
    if (rc) return rc;
    for (int i = 0; i < n; ++i)
        if (envs[i] < 0 || envs[i] >= h->E) { h->setError("mv_draw_cameras: env " + std::to_string(envs[i]) + " out of range"); return MV_ERR_ARG; }
    rc = h->drawCameras(envs, views16, n, w, hgt, want_depth != 0, want_seg != 0);
    if (rc) return rc;
    if (obs) *obs = h->cams.h_obs.p;
    if (depth) *depth = want_depth ? h->cams.h_depth.p : nullptr;
    if (seg) *seg = want_seg ? h->cams.h_seg.p : nullptr;
    if (out_of_range) *out_of_range = *h->cams.h_range.p;
    return MV_OK;
}

int mv_draw_cameras_device(mv_handle h, const int32_t *d_envs, const float *d_views16, int n, int w, int hgt, uint8_t *d_obs, float *d_depth,
                           uint16_t *d_seg, uint32_t **d_out_of_range) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const int rc = cameraCall(h, d_envs, d_views16, n, w, hgt, "mv_draw_cameras_device");
    if (rc) return rc;
    if (n > 0 && !d_obs) { h->setError("mv_draw_cameras_device: null obs buffer"); return MV_ERR_ARG; }
    const int rcl = h->launchCameras(d_envs, d_views16, n, w, hgt, d_obs, d_depth, d_seg);
    if (rcl) return rcl;
    if (d_out_of_range) *d_out_of_range = h->cams.d_range.p;
    return MV_OK;
}

int mv_views_device(mv_handle h, float **d_views) { if (!h || !d_views) return MV_ERR_ARG; *d_views = h->d_views.p; return MV_OK; }

int mv_level_bounds(mv_handle h, float *out6) {
    if (!h || !out6) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    if (!h->didReset) { h->setError("mv_level_bounds before mv_reset"); return MV_ERR_STATE; }
    for (int e = 0; e < h->E; ++e) h->levelBounds(e, out6 + size_t(e) * 6);
    return MV_OK;
}

// ------------------------------------------------------------------------------------------------ state stores
static int statesCallState(mv_handle h, const char *fn) {
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    if (h->hostStepPending) { h->setError(std::string(fn) + ": mv_step_begin is outstanding, call mv_step_end first"); return MV_ERR_STATE; }
    return MV_OK;
}
static StateStore *findStore(mv_handle h, int store, const char *fn) {
    if (store < 0 || store >= int(h->stores.size()) || !h->stores[size_t(store)]) { h->setError(std::string(fn) + ": no state store " + std::to_string(store)); return nullptr; }
    return h->stores[size_t(store)].get();
}
// envs[i] in [0, E), rows[i] in [0, rows), and no destination twice: envs of a load (uniqueEnvs), rows of a save
static int checkStatePairs(mv_handle h, const StateStore &st, const int32_t *envs, const int32_t *rows, int n, bool uniqueEnvs, const char *fn) {
    if (n < 0 || (n > 0 && (!envs || !rows))) { h->setError(std::string(fn) + ": bad env / row arrays"); return MV_ERR_ARG; }
    std::vector<uint8_t> seen(size_t(uniqueEnvs ? h->E : st.rows), 0);
    for (int i = 0; i < n; ++i) {
        if (envs[i] < 0 || envs[i] >= h->E) { h->setError(std::string(fn) + ": env " + std::to_string(envs[i]) + " out of range"); return MV_ERR_ARG; }
        if (rows[i] < 0 || rows[i] >= st.rows) { h->setError(std::string(fn) + ": row " + std::to_string(rows[i]) + " out of range"); return MV_ERR_ARG; }
        const int d = uniqueEnvs ? envs[i] : rows[i];
        if (seen[size_t(d)]++) { h->setError(std::string(fn) + (uniqueEnvs ? ": env " : ": row ") + std::to_string(d) + " is a destination twice"); return MV_ERR_ARG; }
    }
    return MV_OK;
}

int mv_states_create(mv_handle h, int rows, int *store) {
    if (!store) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_states_create");
    if (rc) return rc;
    if (rows < 1) { h->setError("mv_states_create: rows must be positive"); return MV_ERR_ARG; }
    return h->statesCreate(rows, store);
}

int mv_states_save(mv_handle h, int store, const int32_t *envs, const int32_t *rows, int n) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_states_save");
    if (rc) return rc;
    StateStore *st = findStore(h, store, "mv_states_save");
    if (!st) return MV_ERR_ARG;
    rc = checkStatePairs(h, *st, envs, rows, n, false, "mv_states_save");
    if (rc || n == 0) return rc;
    return h->statesSave(*st, envs, rows, n);
}

int mv_states_load(mv_handle h, int store, const int32_t *rows, const int32_t *envs, int n) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_states_load");
    if (rc) return rc;
    StateStore *st = findStore(h, store, "mv_states_load");
    if (!st) return MV_ERR_ARG;
    rc = checkStatePairs(h, *st, envs, rows, n, true, "mv_states_load");
    if (rc || n == 0) return rc;
    for (int i = 0; i < n; ++i) {
        const StateStore::HostRow &r = st->host[size_t(rows[i])];
        if (!r.saved) { h->setError("mv_states_load: row " + std::to_string(rows[i]) + " was never saved"); return MV_ERR_ARG; }
        // the generator travels by value and the reward-shaping row stays with the env: a row of another scenario would turn the env into
        // that scenario with a reward table that does not fit it
        if (r.scenario != h->envScenarioName[size_t(envs[i])]) {
            h->setError("mv_states_load: row " + std::to_string(rows[i]) + " holds a " + r.scenario + " env, env " + std::to_string(envs[i]) + " runs " +
                        h->envScenarioName[size_t(envs[i])]);
            return MV_ERR_ARG;
        }
        // level set: the env's bank row must still hold the level the env was saved on, and stay pickable for its next episodes' probes
        if (r.bankRow >= 0 && (h->rowSeed[size_t(r.bankRow)] != r.bankSeed || h->rowRetiring[size_t(r.bankRow)])) {
            h->setError("mv_states_load: row " + std::to_string(rows[i]) + " was saved on bank row " + std::to_string(r.bankRow) + " (seed " +
                        std::to_string(r.bankSeed) + "), which " + (h->rowRetiring[size_t(r.bankRow)] ? "is being replaced" : "now holds seed " + std::to_string(h->rowSeed[size_t(r.bankRow)])));
            return MV_ERR_ARG;
        }
    }
    return h->statesLoad(*st, rows, envs, n);
}

int mv_reset_envs(mv_handle h, const int32_t *envs, const int32_t *seeds, int n) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_reset_envs");
    if (rc) return rc;
    if (n < 0 || (n > 0 && !envs)) { h->setError("mv_reset_envs: bad env array"); return MV_ERR_ARG; }
    std::vector<uint8_t> seen(size_t(h->E), 0);
    for (int i = 0; i < n; ++i) {
        if (envs[i] < 0 || envs[i] >= h->E) { h->setError("mv_reset_envs: env " + std::to_string(envs[i]) + " out of range"); return MV_ERR_ARG; }
        if (seen[size_t(envs[i])]++) { h->setError("mv_reset_envs: env " + std::to_string(envs[i]) + " is listed twice"); return MV_ERR_ARG; }
    }
    if (n == 0) return MV_OK;
    return h->resetEnvs(envs, seeds, n);
}

int mv_step_envs(mv_handle h, const int32_t *envs, int n) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_step_envs");
    if (rc) return rc;
    if (n < 0 || (n > 0 && !envs)) { h->setError("mv_step_envs: bad env array"); return MV_ERR_ARG; }
    // the list becomes the active mask in pinned memory (the previous call's upload has finished: the call is synchronous)
    uint8_t *mask = h->h_active.p;
    std::memset(mask, 0, size_t(h->E));
    for (int i = 0; i < n; ++i) {
        if (envs[i] < 0 || envs[i] >= h->E) { h->setError("mv_step_envs: env " + std::to_string(envs[i]) + " out of range"); return MV_ERR_ARG; }
        if (mask[envs[i]]++) { h->setError("mv_step_envs: env " + std::to_string(envs[i]) + " is listed twice"); return MV_ERR_ARG; }
    }
    if (cudaMemcpyAsync(h->d_active.p, mask, size_t(h->E), cudaMemcpyHostToDevice, h->stream) != cudaSuccess) { h->setError("active mask upload failed"); return MV_ERR_CUDA; }
    return h->stepHost(h->d_active.p);
}

int mv_states_destroy(mv_handle h, int store) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    StateStore *st = findStore(h, store, "mv_states_destroy");
    if (!st) return MV_ERR_ARG;
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { h->setError("stream sync failed"); return MV_ERR_CUDA; }
    h->stores[size_t(store)].reset();
    return MV_OK;
}

int mv_state_row_bytes(mv_handle h, int64_t *out) {
    if (!h || !out) return MV_ERR_ARG;
    *out = int64_t(h->stateRowBytes());
    return MV_OK;
}

// ------------------------------------------------------------------------------------------------ level sets
static int levelSetCall(mv_handle h, const char *fn) {
    if (!h->levelSet) { h->setError(std::string(fn) + ": option level_set is off"); return MV_ERR_STATE; }
    return MV_OK;
}
int mv_level_ids(mv_handle h, const int32_t **out) {
    if (!h || !out) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    const int rc = levelSetCall(h, "mv_level_ids");
    if (rc == MV_OK) *out = h->h_levelIds.p;
    return rc;
}
int mv_level_ids_device(mv_handle h, int32_t **p) {
    if (!h || !p) return MV_ERR_ARG;
    const int rc = levelSetCall(h, "mv_level_ids_device");
    if (rc == MV_OK) *p = h->d_levelIds.p;
    return rc;
}
int mv_next_levels_device(mv_handle h, int32_t **p) {
    if (!h || !p) return MV_ERR_ARG;
    const int rc = levelSetCall(h, "mv_next_levels_device");
    if (rc == MV_OK) *p = h->d_nextLevels.p;
    return rc;
}
int mv_set_next_levels(mv_handle h, const int32_t *envs, const int32_t *levels, int n) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const int rc = levelSetCall(h, "mv_set_next_levels");
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!envs || !levels))) { h->setError("mv_set_next_levels: bad env / level arrays"); return MV_ERR_ARG; }
    for (int i = 0; i < n; ++i) {
        if (envs[i] < 0 || envs[i] >= h->E) { h->setError("mv_set_next_levels: env " + std::to_string(envs[i]) + " out of range"); return MV_ERR_ARG; }
        if (levels[i] < 0 || levels[i] >= h->levelSet) { h->setError("mv_set_next_levels: level " + std::to_string(levels[i]) + " is outside the set of " + std::to_string(h->levelSet)); return MV_ERR_ARG; }
    }
    return n ? h->setNextLevels(envs, levels, n) : MV_OK;
}
uint32_t mv_level_set_pick(uint32_t pick_seed, int32_t episode, int32_t count) { return mvLevelSetPick(pick_seed, episode, count); }

int mv_replace_levels(mv_handle h, const int32_t *rows, const int32_t *seeds, int n) {
    if (!h) return MV_ERR_ARG;
    int rc = levelSetCall(h, "mv_replace_levels");
    if (rc) return rc;
    MV_NOT_IN_STREAM_MODE(h, "mv_replace_levels")
    if ((rc = statesCallState(h, "mv_replace_levels"))) return rc;
    if (n < 0 || (n > 0 && (!rows || !seeds))) { h->setError("mv_replace_levels: bad row / seed arrays"); return MV_ERR_ARG; }
    const size_t B = h->levelRows();
    std::vector<uint8_t> asked(B, 0);
    std::vector<int> pickable(size_t(h->numBanks), 0);
    for (size_t r = 0; r < B; ++r) pickable[r / size_t(h->levelSet)] += h->rowRetiring[r] ? 0 : 1;
    for (int i = 0; i < n; ++i) {
        const int r = rows[i];
        if (r < 0 || size_t(r) >= B) { h->setError("mv_replace_levels: row " + std::to_string(r) + " is outside the bank of " + std::to_string(B)); return MV_ERR_ARG; }
        if (asked[size_t(r)]++) { h->setError("mv_replace_levels: row " + std::to_string(r) + " is listed twice"); return MV_ERR_ARG; }
        if (h->rowRetiring[size_t(r)]) { h->setError("mv_replace_levels: row " + std::to_string(r) + " is already being replaced"); return MV_ERR_ARG; }
        if (--pickable[size_t(r / h->levelSet)] == 0) {
            h->setError("mv_replace_levels: row " + std::to_string(r) + " would leave bank " + std::to_string(r / h->levelSet) + " with no pickable row");
            return MV_ERR_ARG;
        }
    }
    h->replaceLevels(rows, seeds, n);
    return MV_OK;
}

int mv_level_rows(mv_handle h, const int32_t **seeds, const uint8_t **retiring) {
    if (!h || !seeds || !retiring) return MV_ERR_ARG;
    const int rc = levelSetCall(h, "mv_level_rows");
    if (rc) return rc;
    if (!h->didReset) { h->setError("mv_level_rows before mv_reset"); return MV_ERR_STATE; }
    *seeds = h->rowSeed.data();
    *retiring = h->rowRetiring.data();
    return MV_OK;
}

int mv_fetch_obs(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    if (h->hostStepPending) { const int rcp = h->stepEnd(); if (rcp) return rcp; }
    const int rc = h->drain();
    if (rc) return rc;
    const size_t px = size_t(h->N) * h->W * h->H;
    if (h->wantFinal && h->finalOnDevice) {  // terminal frames of mv_step_device steps (host-facing steps store theirs into the host buffer)
        if (cudaMemcpyAsync(h->h_finalObs.p, h->d_finalObs.p, px * 4, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess) { h->setError("final obs download failed"); return MV_ERR_CUDA; }
        if (h->wantDepth && cudaMemcpyAsync(h->h_finalDepth.p, h->d_finalDepth.p, px * sizeof(float), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess) { h->setError("final depth download failed"); return MV_ERR_CUDA; }
    }
    // the state tensors (live and terminal rows): always current in HBM
    if (h->wantState && h->didReset &&
        cudaMemcpyAsync(h->h_state.p, h->d_state.p, sizeof(float) * h->stateBlockFloats(), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess) {
        h->setError("state tensor download failed");
        return MV_ERR_CUDA;
    }
    // the rays (live and terminal): always current in HBM
    if (h->nRays && h->didReset && h->downloadRays(h->stream) != MV_OK) { h->setError("ray download failed"); return MV_ERR_CUDA; }
    // the reward components (step and episode rows): always current in HBM
    if (h->wantRC && h->didReset && h->downloadRC(h->stream) != MV_OK) { h->setError("reward component download failed"); return MV_ERR_CUDA; }
    // after a zero-copy host-facing step the host buffer holds the newer frames: no copy.  Rows copied from a caller's tensor are not the
    // engine's to vouch for: the next step with an active set draws every view again
    if (h->deviceObsFresh) {
        const int rcd = h->downloadViews(0, h->N, h->stream);
        if (rcd) return rcd;
        h->hostObsFresh = h->ownDeviceObsFresh && h->ownDeviceBuffers();
    }
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { h->setError("stream sync failed"); return MV_ERR_CUDA; }
    return MV_OK;
}

int mv_debug_step_profile(mv_handle h, uint32_t *out, int enable) {
    MV_ON_DEVICE(h)
    MV_NOT_IN_STREAM_MODE(h, "mv_debug_step_profile")
    cudaStreamSynchronize(h->stream);
    if (enable && !h->d_prof.p) {
        if (h->d_prof.alloc(size_t(h->E) * 16) != cudaSuccess) { h->setError("profile buffer allocation failed"); return MV_ERR_CUDA; }
        cudaMemset(h->d_prof.p, 0, sizeof(uint32_t) * size_t(h->E) * 16);
    }
    if (out && h->d_prof.p && cudaMemcpy(out, h->d_prof.p, sizeof(uint32_t) * size_t(h->E) * 16, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (!enable) h->d_prof.free();
    return MV_OK;
}

int mv_sync(mv_handle h) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const int rc = h->drain();
    if (rc) return rc;
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { h->setError("stream sync failed"); return MV_ERR_CUDA; }
    h->readKernelTimes();
    return MV_OK;
}

int mv_obs_host(mv_handle h, const uint8_t **out) { if (!h || !out) return MV_ERR_ARG; *out = h->h_obs.p; return MV_OK; }
int mv_depth_host(mv_handle h, const float **out) { if (!h || !out || !h->wantDepth) return MV_ERR_ARG; *out = h->h_depth.p; return MV_OK; }
int mv_segmentation_host(mv_handle h, const uint16_t **out) {
    if (!h || !out) return MV_ERR_ARG;
    if (!h->wantSeg) { h->setError("mv_segmentation_host: option segmentation is off"); return MV_ERR_ARG; }
    *out = h->h_seg.p;
    return MV_OK;
}
int mv_rewards(mv_handle h, const float **out) { if (!h || !out) return MV_ERR_ARG; MV_SYNC_POINT(h) *out = h->h_rewards.p; return MV_OK; }
int mv_dones(mv_handle h, const uint8_t **out) { if (!h || !out) return MV_ERR_ARG; MV_SYNC_POINT(h) *out = h->h_dones.p; return MV_OK; }
int mv_true_objectives(mv_handle h, const float **out) { if (!h || !out) return MV_ERR_ARG; MV_SYNC_POINT(h) *out = h->h_trueObj.p; return MV_OK; }
int mv_done_reasons(mv_handle h, const uint8_t **out) { if (!h || !out) return MV_ERR_ARG; MV_SYNC_POINT(h) *out = h->h_doneReasons.p; return MV_OK; }
static int awaitingBuffer(mv_handle h, const char *fn) {
    if (!h->autoreset) { h->setError(std::string(fn) + ": option autoreset is 0 (no env ever awaits a reset)"); return MV_ERR_ARG; }
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    return MV_OK;
}
int mv_awaiting_reset_host(mv_handle h, const uint8_t **out) {
    if (!h || !out) return MV_ERR_ARG;
    if (const int rc = awaitingBuffer(h, "mv_awaiting_reset_host")) return rc;
    MV_SYNC_POINT(h)
    *out = h->h_awaiting.p;
    return MV_OK;
}
int mv_awaiting_reset_device(mv_handle h, uint8_t **d) {
    if (!h || !d) return MV_ERR_ARG;
    if (const int rc = awaitingBuffer(h, "mv_awaiting_reset_device")) return rc;
    *d = h->d_awaiting.p;
    return MV_OK;
}
static int finalBuffer(mv_handle h, bool depth, const char *fn) {
    if (!h->wantFinal || (depth && !h->wantDepth)) { h->setError(std::string(fn) + ": option final_obs" + (depth ? " and option depth are" : " is") + " off"); return MV_ERR_ARG; }
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    return MV_OK;
}
int mv_final_obs_host(mv_handle h, const uint8_t **out) {
    if (!h || !out) return MV_ERR_ARG;
    const int rc = finalBuffer(h, false, "mv_final_obs_host");
    if (rc == MV_OK) *out = h->h_finalObs.p;
    return rc;
}
int mv_final_depth_host(mv_handle h, const float **out) {
    if (!h || !out) return MV_ERR_ARG;
    const int rc = finalBuffer(h, true, "mv_final_depth_host");
    if (rc == MV_OK) *out = h->h_finalDepth.p;
    return rc;
}
int mv_final_obs_device(mv_handle h, uint8_t **p) {
    if (!h || !p) return MV_ERR_ARG;
    const int rc = finalBuffer(h, false, "mv_final_obs_device");
    if (rc == MV_OK) *p = h->d_finalObs.p;
    return rc;
}
int mv_final_depth_device(mv_handle h, float **p) {
    if (!h || !p) return MV_ERR_ARG;
    const int rc = finalBuffer(h, true, "mv_final_depth_device");
    if (rc == MV_OK) *p = h->d_finalDepth.p;
    return rc;
}
// option state_tensors (and final_obs, for the terminal rows) is on and the engine reset
static int stateTensorCall(mv_handle h, bool terminal, const char *fn) {
    if (!h) return MV_ERR_ARG;
    if (!h->wantState || (terminal && !h->wantFinal)) {
        h->setError(std::string(fn) + ": option state_tensors" + (terminal ? " or option final_obs is" : " is") + " off");
        return MV_ERR_ARG;
    }
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    return MV_OK;
}
// the four tensors of the live or terminal rows in `block` into the non-null outs
static void stateTensorOuts(mv_handle h, float *block, bool terminal, float **agents, float **envs, float **objects, float **rewards) {
    float **outs[4] = {agents, envs, objects, rewards};
    for (int k = 0; k < 4; ++k)
        if (outs[k]) *outs[k] = h->stateTensor(block, k, terminal);
}
int mv_state_tensors_host(mv_handle h, const float **agents, const float **envs, const float **objects, const float **rewards) {
    const int rc = stateTensorCall(h, false, "mv_state_tensors_host");
    if (rc == MV_OK) stateTensorOuts(h, h->h_state.p, false, const_cast<float **>(agents), const_cast<float **>(envs), const_cast<float **>(objects), const_cast<float **>(rewards));
    return rc;
}
int mv_state_tensors_device(mv_handle h, float **agents, float **envs, float **objects, float **rewards) {
    const int rc = stateTensorCall(h, false, "mv_state_tensors_device");
    if (rc == MV_OK) stateTensorOuts(h, h->d_state.p, false, agents, envs, objects, rewards);
    return rc;
}
int mv_final_state_tensors_host(mv_handle h, const float **agents, const float **envs, const float **objects, const float **rewards) {
    const int rc = stateTensorCall(h, true, "mv_final_state_tensors_host");
    if (rc == MV_OK) stateTensorOuts(h, h->h_state.p, true, const_cast<float **>(agents), const_cast<float **>(envs), const_cast<float **>(objects), const_cast<float **>(rewards));
    return rc;
}
int mv_final_state_tensors_device(mv_handle h, float **agents, float **envs, float **objects, float **rewards) {
    const int rc = stateTensorCall(h, true, "mv_final_state_tensors_device");
    if (rc == MV_OK) stateTensorOuts(h, h->d_state.p, true, agents, envs, objects, rewards);
    return rc;
}
// option reward_components is on and the engine reset
static int rewardComponentCall(mv_handle h, const char *fn) {
    if (!h) return MV_ERR_ARG;
    if (!h->wantRC) { h->setError(std::string(fn) + ": option reward_components is off"); return MV_ERR_ARG; }
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    return MV_OK;
}
int mv_reward_components_host(mv_handle h, const float **step, const float **episode) {
    const int rc = rewardComponentCall(h, "mv_reward_components_host");
    if (rc == MV_OK) { if (step) *step = h->rcTensor(h->h_rc.p, 0); if (episode) *episode = h->rcTensor(h->h_rc.p, 1); }
    return rc;
}
int mv_reward_components_device(mv_handle h, float **step, float **episode) {
    const int rc = rewardComponentCall(h, "mv_reward_components_device");
    if (rc == MV_OK) { if (step) *step = h->rcTensor(h->d_rc.p, 0); if (episode) *episode = h->rcTensor(h->d_rc.p, 1); }
    return rc;
}
int mv_reward_component_keys(const char *scenario, const char **keys8) {
    if (!scenario || !keys8) return MV_ERR_ARG;
    const int sc = mv::scenarioFromName(scenario);
    if (sc < 0) return MV_ERR_ARG;
    for (int k = 0; k < MV_R_COUNT; ++k) keys8[k] = mv::rewardKey(sc, k);
    return MV_OK;
}
int mv_set_rays(mv_handle h, const float *dirs3, int n, float max_dist) {
    if (!h) return MV_ERR_ARG;
    if (h->didReset) { h->setError("mv_set_rays must be called before the first reset"); return MV_ERR_STATE; }
    if (n < 0 || n > MV_MAX_RAYS) { h->setError("mv_set_rays: n out of range [0, MV_MAX_RAYS]"); return MV_ERR_ARG; }
    if (n > 0 && !dirs3) { h->setError("mv_set_rays: null directions"); return MV_ERR_ARG; }
    if (!std::isfinite(max_dist) || !(max_dist > 0.0f)) { h->setError("mv_set_rays: max_dist must be finite and > 0"); return MV_ERR_ARG; }
    for (int i = 0; i < n; ++i) {
        const float *d = dirs3 + 3 * i;
        if (!std::isfinite(d[0]) || !std::isfinite(d[1]) || !std::isfinite(d[2]) || (d[0] == 0.0f && d[1] == 0.0f && d[2] == 0.0f)) {
            h->setError("mv_set_rays: direction " + std::to_string(i) + " is zero or not finite");
            return MV_ERR_ARG;
        }
    }
    h->rayDirs.assign(dirs3, dirs3 + 3 * size_t(n));
    h->nRays = n;
    h->rayMaxDist = max_dist;
    return MV_OK;
}
// the rays are on (and, for the terminal rays, option final_obs) and the engine reset
static int rayCall(mv_handle h, bool terminal, const char *fn) {
    if (!h) return MV_ERR_ARG;
    if (!h->nRays || (terminal && !h->wantFinal)) {
        h->setError(std::string(fn) + (terminal ? ": the rays or option final_obs are off" : ": the rays are off"));
        return MV_ERR_ARG;
    }
    if (!h->didReset) { h->setError(std::string(fn) + " before mv_reset"); return MV_ERR_STATE; }
    return MV_OK;
}
int mv_rays_host(mv_handle h, const float **dist, const uint16_t **tag) {
    const int rc = rayCall(h, false, "mv_rays_host");
    if (rc == MV_OK) { if (dist) *dist = h->h_rayDist.p; if (tag) *tag = h->h_rayTag.p; }
    return rc;
}
int mv_rays_device(mv_handle h, float **dist, uint16_t **tag) {
    const int rc = rayCall(h, false, "mv_rays_device");
    if (rc == MV_OK) { if (dist) *dist = h->d_rayDist.p; if (tag) *tag = h->d_rayTag.p; }
    return rc;
}
int mv_final_rays_host(mv_handle h, const float **dist, const uint16_t **tag) {
    const int rc = rayCall(h, true, "mv_final_rays_host");
    if (rc == MV_OK) { if (dist) *dist = h->h_rayDist.p + h->rayCount(); if (tag) *tag = h->h_rayTag.p + h->rayCount(); }
    return rc;
}
int mv_final_rays_device(mv_handle h, float **dist, uint16_t **tag) {
    const int rc = rayCall(h, true, "mv_final_rays_device");
    if (rc == MV_OK) { if (dist) *dist = h->d_rayDist.p + h->rayCount(); if (tag) *tag = h->d_rayTag.p + h->rayCount(); }
    return rc;
}
int mv_set_obs_buffer(mv_handle h, uint8_t *d_obs, float *d_depth) {
    MV_ON_DEVICE(h)
    // the pointer is a launch parameter: steps already enqueued keep writing the previous buffer, the next step writes the new one.  No
    // synchronisation here (a consumer that double-buffers its tensor switches every step); mv_sync before freeing a buffer.
    h->obsOut = d_obs ? d_obs : h->d_obs.p;
    h->depthOut = d_depth ? d_depth : h->d_depth.p;
    return MV_OK;
}
int mv_actions_device(mv_handle h, int32_t **p) { if (!h || !p) return MV_ERR_ARG; *p = h->d_actions.p; return MV_OK; }
int mv_obs_device(mv_handle h, uint8_t **p) {
    if (!h || !p) return MV_ERR_ARG;
    if (h->didReset && !h->deviceObsFresh) { h->setError("the last step delivered its frames to the host buffer only (zero-copy): the HBM tensor is stale; use mv_step_device or option zero_copy=0"); return MV_ERR_STATE; }
    *p = h->obsOut;
    return MV_OK;
}
int mv_depth_device(mv_handle h, float **p) {
    if (!h || !p || !h->wantDepth) return MV_ERR_ARG;
    if (h->didReset && !h->deviceObsFresh) { h->setError("the last step delivered its frames to the host buffer only (zero-copy): the HBM tensor is stale"); return MV_ERR_STATE; }
    *p = h->depthOut;
    return MV_OK;
}
int mv_segmentation_device(mv_handle h, uint16_t **p) {
    if (!h || !p) return MV_ERR_ARG;
    if (!h->wantSeg) { h->setError("mv_segmentation_device: option segmentation is off"); return MV_ERR_ARG; }
    if (h->didReset && !h->deviceObsFresh) { h->setError("the last step delivered its frames to the host buffer only (zero-copy): the HBM tensor is stale"); return MV_ERR_STATE; }
    *p = h->d_seg.p;
    return MV_OK;
}
int mv_rewards_device(mv_handle h, float **p) { if (!h || !p) return MV_ERR_ARG; *p = h->d_rewards.p; return MV_OK; }
int mv_dones_device(mv_handle h, uint8_t **p) { if (!h || !p) return MV_ERR_ARG; *p = h->d_dones.p; return MV_OK; }
int mv_done_reasons_device(mv_handle h, uint8_t **p) { if (!h || !p) return MV_ERR_ARG; *p = h->d_doneReasons.p; return MV_OK; }
int mv_true_objectives_device(mv_handle h, float **p) { if (!h || !p) return MV_ERR_ARG; *p = h->d_trueObj.p; return MV_OK; }
int mv_stream(mv_handle h, void **s) { if (!h || !s) return MV_ERR_ARG; *s = h->stream; return MV_OK; }

int mv_get_reward_shaping(mv_handle h, int env, int agent, const char **keys, float *vals, int cap, int *n) {
    if (!h || env < 0 || env >= h->E || agent < 0 || agent >= h->A || !n) return MV_ERR_ARG;
    auto &rs = h->shaping[size_t(env) * h->A + agent];
    *n = int(rs.size());
    for (int i = 0; i < int(rs.size()) && i < cap; ++i) { keys[i] = rs[size_t(i)].first.c_str(); vals[i] = rs[size_t(i)].second; }
    return MV_OK;
}

int mv_set_reward_shaping(mv_handle h, int env, int agent, const char *const *keys, const float *vals, int n) {
    if (!h || env < 0 || env >= h->E || agent < 0 || agent >= h->A) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    // Scenario::setRewardShaping replaces the whole map (scenario.hpp:215); a scheme lacking a key the scenario reads
    // makes the reference throw std::out_of_range at the next reward event (scenario.hpp:253) -> reject it up front
    std::map<std::string, float> m;
    for (int i = 0; i < n; ++i) m[keys[i]] = vals[i];
    for (auto &kv : mv::defaultRewardShaping(h->envScenarioName[size_t(env)]))  // the keys of this env's scenario
        if (!m.count(kv.first)) { h->setError("reward shaping lacks key " + kv.first + " of env " + std::to_string(env) + "'s scenario " + h->envScenarioName[size_t(env)]); return MV_ERR_ARG; }
    const size_t view = size_t(env) * h->A + agent;
    h->shaping[view].assign(m.begin(), m.end());
    h->fillRtableRow(int(view));
    h->rtableDirty = true;
    if (!h->streamMode) return MV_OK;
    // in stream mode at once, on the engine's device: a host-path step may never come
    DeviceGuard dg(h->device);
    if (!dg.ok) { h->setError("cudaSetDevice failed"); return MV_ERR_CUDA; }
    return h->uploadRtable();
}

int mv_faults(mv_handle h, int32_t *out) {
    if (!out) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    if (h->stream) cudaStreamSynchronize(h->stream);
    std::vector<MvEnvState> st(size_t(h->E));
    if (cudaMemcpy(st.data(), h->d_envs.p, sizeof(MvEnvState) * st.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (cudaMemcpy(h->h_faults.p, h->d_faults.p, sizeof(int32_t) * h->E, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    int32_t f = 0;
    for (int e = 0; e < h->E; ++e) f |= st[size_t(e)].faults | h->h_faults.p[e];
    *out = f;
    return MV_OK;
}
// totals since enable: {work items, instances read, instances with visible items, items, clipped items, triangles, batches, -}
int mv_debug_raster_stats(mv_handle h, unsigned long long *out16, int enable) {
    MV_ON_DEVICE(h)
    MV_NOT_IN_STREAM_MODE(h, "mv_debug_raster_stats")
    cudaStreamSynchronize(h->stream);
    if (out16 && h->d_rasterStats.p && cudaMemcpy(out16, h->d_rasterStats.p, 128, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (enable && !h->d_rasterStats.p) {
        if (h->d_rasterStats.alloc(16) != cudaSuccess) { h->setError("raster stats allocation failed"); return MV_ERR_CUDA; }
    }
    if (enable) cudaMemset(h->d_rasterStats.p, 0, 128);
    else h->d_rasterStats.free();
    return MV_OK;
}
int mv_debug_static_cap(mv_handle h) { return h ? h->levels.staticCap : MV_ERR_ARG; }  // current size of the per-level static-box arrays
int mv_debug_raster_config(mv_handle h, int32_t *out4) {  // {persistent grid, CTAs per SM, dynamic shared memory bytes, row bands per view}
    if (!h || !out4) return MV_ERR_ARG;
    out4[0] = h->rasterGrid; out4[1] = h->rasterCtasPerSM; out4[2] = int32_t(h->rasterSmem); out4[3] = h->rasterBands;
    return MV_OK;
}
int mv_fault_word(mv_handle h, int32_t *out) {  // no device round trip: the step kernel ORs raised bits into pinned host memory
    if (!h || !out) return MV_ERR_ARG;
    *out = *const_cast<volatile int32_t *>(h->h_faultWord.p);
    return MV_OK;
}
int mv_kernel_launches(mv_handle h, int64_t *out) { if (!h || !out) return MV_ERR_ARG; *out = h->launches; return MV_OK; }
int mv_last_kernel_ms(mv_handle h, float *out2) { if (!h || !out2) return MV_ERR_ARG; out2[0] = h->lastMs[0]; out2[1] = h->lastMs[1]; return MV_OK; }
int mv_last_final_ms(mv_handle h, float *out) { if (!h || !out) return MV_ERR_ARG; *out = h->lastFinalMs; return MV_OK; }
int mv_last_rays_ms(mv_handle h, float *out) { if (!h || !out) return MV_ERR_ARG; *out = h->lastRaysMs; return MV_OK; }

int mv_close(mv_handle h) {
    if (!h) return MV_ERR_ARG;
    DeviceGuard dg__(h->device);  // not MV_ON_DEVICE: the engine is freed even when the switch fails
    if (h->streamMode) cudaDeviceSynchronize();  // graph replays on the caller's streams may still use the engine's buffers
    delete h;
    return MV_OK;
}

// ------------------------------------------------------------------------------------------------ introspection (tests)
// the mv_debug_get_level layout of level L (with its static boxes and their rotations) for A agents; `spawnBasis` appends the agents'
// spawn yaw bases as float bits
static int dumpLevel(const MvLevel &L, const MvBox *statics, const float *staticRot, int A, bool spawnBasis, int32_t *out, int cap) {
    std::vector<int32_t> o;
    o.push_back(L.n_grid_static); o.push_back(L.n_terrain); o.push_back(L.n_obj);
    for (int a = 0; a < 3; ++a) o.push_back(L.bz_min[a]);
    for (int a = 0; a < 3; ++a) o.push_back(L.bz_max[a]);
    for (int i = 0; i < L.n_grid_static; ++i) {
        const MvBox &b = statics[i];
        // invert centre/half back to inclusive voxel bounds: min = c - h, max = c + h - 1
        const float vs = L.scenario == MV_SCENARIO_SOKOBAN ? 2.0f : 1.0f;  // voxel size of the scenario's grid
        for (int a = 0; a < 3; ++a) o.push_back(int(lroundf((b.c[a] - b.h[a]) / vs)));
        for (int a = 0; a < 3; ++a) o.push_back(int(lroundf((b.c[a] + b.h[a]) / vs)) - 1);
        o.push_back(b.flags & 255); o.push_back(int(kPaletteRgb[b.color]));
    }
    for (int i = 0; i < L.n_terrain; ++i) {
        o.push_back(L.terrain[i].type);
        for (int a = 0; a < 6; ++a) o.push_back(L.terrain[i].bb[a]);
    }
    for (int i = 0; i < L.n_obj; ++i) for (int a = 0; a < 3; ++a) o.push_back(L.obj_init[i].voxel[a]);
    for (int i = 0; i < A; ++i) for (int a = 0; a < 3; ++a) o.push_back(int(L.init_pos[i][a]));
    if (L.scenario != MV_SCENARIO_TOWER) {
        o.push_back(L.n_movable);  // numPlatforms
        // reward-object voxels; for the hexagonal mazes the free-standing colliders instead (bit patterns of centre, half extents, orientation)
        const bool hex = L.scenario == MV_SCENARIO_HEX_EXPLORE || L.scenario == MV_SCENARIO_HEX_MEMORY || L.scenario == MV_SCENARIO_EMPTY;
        o.push_back(hex ? 0 : L.n_reward);
        for (int i = 0; i < L.n_reward && !hex; ++i) for (int a = 0; a < 3; ++a) o.push_back(L.reward_voxel[i][a]);
        if (hex) {
            o.push_back(L.n_static);
            for (int i = 0; i < L.n_static; ++i) {
                const MvBox &b = statics[i];
                const float rot[2] = {(b.flags & MV_ROTATED) ? staticRot[i * 2] : 1.0f, (b.flags & MV_ROTATED) ? staticRot[i * 2 + 1] : 0.0f};
                int32_t w[8];
                std::memcpy(w, b.c, 12); std::memcpy(w + 3, b.h, 12); std::memcpy(w + 6, rot, 8);
                for (int k = 0; k < 8; ++k) o.push_back(w[k]);
            }
        }
    }
    for (int i = 0; i < A && spawnBasis; ++i) for (int k = 0; k < 9; ++k) { int32_t u; std::memcpy(&u, &L.spawn_basis[i][k], 4); o.push_back(u); }
    if (int(o.size()) > cap) return -int(o.size());
    std::memcpy(out, o.data(), o.size() * sizeof(int32_t));
    return int(o.size());
}

int mv_debug_get_level(mv_handle h, int env, int32_t *out, int cap) {
    if (!h || env < 0 || env >= h->E || !h->didReset) return MV_ERR_ARG;
    MV_SYNC_POINT(h)
    const size_t lid = h->liveRow(env);
    return dumpLevel(h->levels.level(lid), h->levels.statics(lid), h->levels.rotations(lid), h->A, false, out, cap);
}

int mv_debug_get_state(mv_handle h, int env, float *out, int cap) {
    if (!h || env < 0 || env >= h->E || !h->didReset) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    MvEnvState es;
    std::vector<MvAgent> ag(size_t(h->A));
    std::vector<MvObject> ob(MV_MAX_OBJECTS);
    cudaStreamSynchronize(h->stream);
    if (cudaMemcpy(&es, &h->d_envs.p[env], sizeof es, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (cudaMemcpy(ag.data(), &h->d_agents.p[size_t(env) * h->A], sizeof(MvAgent) * h->A, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (cudaMemcpy(ob.data(), &h->d_objects.p[size_t(env) * MV_MAX_OBJECTS], sizeof(MvObject) * MV_MAX_OBJECTS, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    const size_t lid = h->rowOfSlot(env, es.slot);
    const MvLevel &L = h->levels.level(lid);
    std::vector<float> o;
    int ncol = h->A + L.n_obj;
    const MvBox *statics = h->levels.statics(lid);
    for (int i = 0; i < L.n_static; ++i) ncol += (statics[i].flags & MV_SOLID) ? 1 : 0;
    const float len = L.episode_len;
    o.push_back(es.episode_sec); o.push_back(len); o.push_back(float(es.num_frames)); o.push_back(float(es.highest_tower));
    o.push_back(es.bz_reward); o.push_back(float(L.n_obj)); o.push_back(float(ncol)); o.push_back(0.f);
    for (int i = 0; i < h->A; ++i) {
        const MvAgent &a = ag[size_t(i)];
        for (int k = 0; k < 3; ++k) o.push_back(a.pos[k]);
        for (int k = 0; k < 9; ++k) o.push_back(a.basis[k]);
        for (int k = 0; k < 3; ++k) o.push_back(a.hvel[k]);
        for (float x : {a.vvel, a.voff, a.step_off, a.was_on_ground ? 1.f : 0.f, a.was_jumping ? 1.f : 0.f, a.jump_speed, a.cur_x, float(a.carrying), a.total_reward,
                        h->h_rewards.p[size_t(env) * h->A + i], 0.f})
            o.push_back(x);
    }
    for (int i = 0; i < L.n_obj; ++i) {
        const MvObject &b = ob[size_t(i)];
        float t[3] = {b.t[0], b.t[1], b.t[2]};
        if (b.parent >= 0) {  // absolute translation of a carried object: ((agent*camera)*pickup)*local, as the oracle reports it
            const MvAgent &a = ag[size_t(b.parent)];
            mvh::M4 objT, cam;
            std::memcpy(&objT.c[0][0], a.object_t, 64); std::memcpy(&cam.c[0][0], a.cam_local, 64);
            const mvh::M4 pick = mvh::mul(mvh::translation(0.0f, -0.44f, -1.0f), mvh::identity());
            const mvh::M4 local = mvh::mul(mvh::translation(b.t[0], b.t[1], b.t[2]), mvh::mul(mvh::scaling(b.s[0], b.s[1], b.s[2]), mvh::identity()));
            const mvh::M4 abs = mvh::mul(mvh::mul(mvh::mul(objT, cam), pick), local);
            t[0] = abs.c[3][0]; t[1] = abs.c[3][1]; t[2] = abs.c[3][2];
        }
        for (float x : {t[0], t[1], t[2], b.s[0], b.s[1], b.s[2], float(b.parent), b.enabled ? 1.f : 0.f, 0.f}) o.push_back(x);
    }
    if (L.scenario != MV_SCENARIO_TOWER) {
        o.push_back(float(es.solved)); o.push_back(float(L.scenario == MV_SCENARIO_HEX_MEMORY ? uint32_t(es.positive_collected) : es.reached_exit));
        for (int w = 0; w < 3; ++w) o.push_back(float(es.reward_alive[w] & 0xffffffu)), o.push_back(float(es.reward_alive[w] >> 24));
    }
    if (int(o.size()) > cap) return -int(o.size());
    std::memcpy(out, o.data(), o.size() * sizeof(float));
    return int(o.size());
}

int mv_debug_get_voxels(mv_handle h, int env, int32_t *out, int cap) {
    if (!h || env < 0 || env >= h->E || !h->didReset) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    MvEnvState es;
    cudaStreamSynchronize(h->stream);
    if (cudaMemcpy(&es, &h->d_envs.p[env], sizeof es, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    const size_t lid = h->rowOfSlot(env, es.slot);
    const MvLevel &L = h->levels.level(lid);
    const uint32_t *sol = h->levels.plane(lid, 0), *exitBits = h->levels.plane(lid, 1), *lavaBits = h->levels.plane(lid, 2);
    const MvBox *statics = h->levels.statics(lid);
    std::vector<uint8_t> og(size_t(h->gridCells));
    if (cudaMemcpy(og.data(), h->d_objGrid.p + size_t(env) * h->gridCells, og.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    std::vector<MvObject> ob(size_t(L.n_obj > 0 ? L.n_obj : 1));
    if (cudaMemcpy(ob.data(), &h->d_objects.p[size_t(env) * MV_MAX_OBJECTS], sizeof(MvObject) * ob.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    // opacity is a property of the box a solid voxel belongs to
    std::vector<std::array<int32_t, 4>> v;
    for (int x = 0; x < L.grid_dim[0]; ++x)
        for (int y = 0; y < L.grid_dim[1]; ++y)
            for (int z = 0; z < L.grid_dim[2]; ++z) {
                const int idx = (x * L.grid_dim[1] + y) * L.grid_dim[2] + z;
                int flags = 0;
                if ((sol[idx >> 5] >> (idx & 31)) & 1u) {
                    flags |= 1;
                    const float vs = L.scenario == MV_SCENARIO_SOKOBAN ? 2.0f : 1.0f;
                    const float cx = (x + L.grid_org[0] + 0.5f) * vs, cy = (y + L.grid_org[1] + 0.5f) * vs, cz = (z + L.grid_org[2] + 0.5f) * vs;
                    for (int i = 0; i < L.n_grid_static; ++i) {
                        const MvBox &b = statics[i];
                        if (fabsf(cx - b.c[0]) < b.h[0] && fabsf(cy - b.c[1]) < b.h[1] && fabsf(cz - b.c[2]) < b.h[2]) { flags |= (b.flags & MV_OPAQUE); break; }
                    }
                }
                if (og[size_t(idx)] != MV_NO_OBJECT) flags |= 4;
                if ((exitBits[idx >> 5] >> (idx & 31)) & 1u) flags |= 1 << 8;
                if ((lavaBits[idx >> 5] >> (idx & 31)) & 1u) flags |= 2 << 8;
                if (flags) v.push_back({x + L.grid_org[0], y + L.grid_org[1], z + L.grid_org[2], flags});
            }
    // objects put down outside the grid live only in their translation (the step kernel's objAt); the scenarios without stacking
    // keep their objects elsewhere (Sokoban's boxes on its 2-unit grid) or in no grid at all
    const bool stacking = L.scenario == MV_SCENARIO_TOWER || L.scenario == MV_SCENARIO_OBSTACLES || L.scenario == MV_SCENARIO_COLLECT || L.scenario == MV_SCENARIO_REARRANGE;
    for (int i = 0; i < L.n_obj && stacking; ++i) {
        const MvObject &b = ob[size_t(i)];
        if (b.parent >= 0) continue;
        const int x = int(std::floor(b.t[0])), y = int(std::floor(b.t[1])), z = int(std::floor(b.t[2]));
        const int gx = x - L.grid_org[0], gy = y - L.grid_org[1], gz = z - L.grid_org[2];
        if (gx < 0 || gy < 0 || gz < 0 || gx >= L.grid_dim[0] || gy >= L.grid_dim[1] || gz >= L.grid_dim[2]) v.push_back({x, y, z, 4});
    }
    std::sort(v.begin(), v.end());
    if (int(v.size()) * 4 > cap) return -int(v.size()) * 4;
    for (size_t i = 0; i < v.size(); ++i) std::memcpy(out + i * 4, v[i].data(), 16);
    return int(v.size()) * 4;
}

int mv_debug_get_instances(mv_handle h, int env, float *out, int cap) {
    if (!h || env < 0 || env >= h->E || !h->didReset) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int32_t cnt[8];
    cudaStreamSynchronize(h->stream);
    if (cudaMemcpy(cnt, h->d_instCounts.p + size_t(env) * 8, 32, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    std::vector<MvInstance> inst(static_cast<size_t>(cnt[1] > 0 ? cnt[1] : 1));
    if (cudaMemcpy(inst.data(), h->d_inst.p + size_t(env) * size_t(h->instCap()), sizeof(MvInstance) * inst.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    if (cnt[1] * 18 > cap) return -cnt[1] * 18;
    for (int i = 0; i < cnt[1]; ++i) {
        out[i * 18] = float(inst[size_t(i)].mesh); out[i * 18 + 1] = float(inst[size_t(i)].color);
        std::memcpy(out + i * 18 + 2, inst[size_t(i)].model, 64);
    }
    return cnt[1] * 18;
}

int mv_debug_get_view(mv_handle h, int env, int agent, float *out16) {
    if (!h || env < 0 || env >= h->E || agent < 0 || agent >= h->A || !h->didReset) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    cudaStreamSynchronize(h->stream);
    if (cudaMemcpy(out16, h->d_views.p + (size_t(env) * h->A + agent) * 16, 64, cudaMemcpyDeviceToHost) != cudaSuccess) return MV_ERR_CUDA;
    return MV_OK;
}

int mv_debug_view_order(mv_handle h, uint32_t *out, int cap) {
    if (!h || !out) return MV_ERR_ARG;
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    const size_t words = h->costItems() + size_t(h->E) + 1;
    if (size_t(cap) < words) return -int(words);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess || cudaMemcpy(out, h->d_viewCost.p, sizeof(uint32_t) * words, cudaMemcpyDeviceToHost) != cudaSuccess) {
        h->setError("mv_debug_view_order: copy failed");
        return MV_ERR_CUDA;
    }
    return int(words);
}

int mv_debug_warp_agent(mv_handle h, int env, int agent, const float pos[3], const float basis9[9]) {
    MV_ON_DEVICE(h)
    MV_SYNC_POINT(h)
    int rc = statesCallState(h, "mv_debug_warp_agent");
    if (rc) return rc;
    if (env < 0 || env >= h->E || agent < 0 || agent >= h->A) { h->setError("mv_debug_warp_agent: env / agent out of range"); return MV_ERR_ARG; }
    if (!pos || !basis9) { h->setError("mv_debug_warp_agent: null pointer"); return MV_ERR_ARG; }
    // MvAgent starts with pos[3], basis[9], hvel[3], vvel: one contiguous 16-float write
    float w[16] = {};
    std::memcpy(w, pos, 12);
    std::memcpy(w + 3, basis9, 36);
    for (int k = 0; k < 12; ++k)
        if (!std::isfinite(w[k])) { h->setError("mv_debug_warp_agent: non-finite value"); return MV_ERR_ARG; }
    return h->warpAgent(env, agent, w);
}

int mv_debug_render_instances_ex(const float *view16, const float *inst18, int n, int w, int h, const int *opts, uint8_t *rgba, float *depth,
                                 uint16_t *seg, unsigned long long *stats) {
    if (!view16 || !inst18 || !opts || !rgba || n < 0 || n > 4096) return MV_ERR_ARG;
    if (w < 32 || h < 4 || w % 32 || h % 4 || w > kMaxRasterWidth || h > 4096) return MV_ERR_ARG;  // what mv_draw_hires accepts
    const bool fast = opts[0] != 0, wantSeg = opts[1] != 0;
    if ((opts[0] | opts[1]) & ~1 || (wantSeg && !seg)) return MV_ERR_ARG;
    const int triCap = opts[2] ? opts[2] : kDefaultTriCap;
    if (triCap < 32 || triCap > mvr::kMaxTriCap) return MV_ERR_ARG;
    // row bands: opts[3] of them (the last one may be shorter), or 0 = the rule of mv_draw_hires (bands of about a hundred tiles)
    int bandRows;
    if (opts[3] == 0) bandRows = hiresBandRows(w);
    else if (opts[3] > 0 && opts[3] <= h / 4) bandRows = ((h / 4 + opts[3] - 1) / opts[3]) * 4;
    else return MV_ERR_ARG;
    const int bands = (h + bandRows - 1) / bandRows;
    int ndev = 0, dev = 0, maxOptin = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&maxOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return MV_ERR_CUDA;
    const size_t smem = mvr::smemLayout(triCap).total;
    if (smem > size_t(maxOptin)) return MV_ERR_ARG;
    // instances must arrive sorted by mesh type, boxes first (draw order); instance i carries segmentation tag i + 1
    std::vector<MvInstance> inst(size_t(n ? n : 1));
    int32_t cnt[8] = {0, n, 0, 0, 0, 0, 0, 0};
    for (int i = 0, last = 0; i < n; ++i) {
        MvInstance &d = inst[size_t(i)];
        d.mesh = int(inst18[i * 18]); d.color = int(inst18[i * 18 + 1]);
        std::memcpy(d.model, inst18 + i * 18 + 2, 64);
        d.pad[0] = i + 1; d.pad[1] = 0;
        if (d.mesh < last || d.mesh > 4 || d.color < 0 || d.color >= 22) return MV_ERR_ARG;
        last = d.mesh;
        cnt[d.mesh == 0 ? 0 : 1 + d.mesh] += 1;
    }
    MvConsts k;
    fillConsts(k, w, h);
    if (uploadPalette() != cudaSuccess) return MV_ERR_CUDA;
    const ViewKernel fn = viewKernelOf(mvr::Items::All, wantSeg, fast);
    DevBuf<MvInstance> dInst; DevBuf<int32_t> dCnt; DevBuf<float> dView, dDepth; DevBuf<uint8_t> dObs; DevBuf<uint16_t> dSeg;
    DevBuf<uint32_t> dCtr; DevBuf<unsigned long long> dSpill, dStats;
    const size_t px = size_t(w) * size_t(h);
    // the attribute is the device maximum, as configureRaster sets it: an engine alive in this process keeps launching with its own tri_cap
    bool ok = dInst.alloc(inst.size()) == cudaSuccess && dCnt.alloc(8) == cudaSuccess && dView.alloc(16) == cudaSuccess &&
              dObs.alloc(px * 4) == cudaSuccess && dDepth.alloc(px) == cudaSuccess && dSeg.alloc(px) == cudaSuccess && dStats.alloc(16) == cudaSuccess &&
              dCtr.alloc(4) == cudaSuccess && dSpill.alloc(size_t(bands) * size_t(w) * bandRows) == cudaSuccess &&
              cudaFuncSetAttribute(reinterpret_cast<const void *>(fn), cudaFuncAttributeMaxDynamicSharedMemorySize, maxOptin) == cudaSuccess;
    if (ok) {
        cudaMemcpy(dInst.p, inst.data(), sizeof(MvInstance) * inst.size(), cudaMemcpyHostToDevice);
        cudaMemcpy(dCnt.p, cnt, 32, cudaMemcpyHostToDevice);
        cudaMemcpy(dView.p, view16, 64, cudaMemcpyHostToDevice);
        cudaMemset(dCtr.p, 0, 16);
        cudaMemset(dStats.p, 0, 16 * sizeof(unsigned long long));
        mvr::ViewParams vp = frameParams(w, h, bands, bandRows, dSpill.p, triCap, k);
        vp.instances = dInst.p; vp.instCounts = dCnt.p; vp.views = dView.p; vp.instStride = int(inst.size()); vp.obs = dObs.p; vp.depth = depth ? dDepth.p : nullptr;
        vp.seg = wantSeg ? dSeg.p : nullptr; vp.stats = stats ? dStats.p : nullptr;
        vp.workCounter = dCtr.p; vp.viewBase = 0; vp.N = 1; vp.A = 1;
        fn<<<bands, mvr::kThreads, smem>>>(vp);
        ok = cudaDeviceSynchronize() == cudaSuccess;
        if (ok) {
            cudaMemcpy(rgba, dObs.p, px * 4, cudaMemcpyDeviceToHost);
            if (depth) cudaMemcpy(depth, dDepth.p, px * 4, cudaMemcpyDeviceToHost);
            if (wantSeg) cudaMemcpy(seg, dSeg.p, px * 2, cudaMemcpyDeviceToHost);
            if (stats) cudaMemcpy(stats, dStats.p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
        }
    }
    return ok ? MV_OK : MV_ERR_CUDA;
}

int mv_debug_render_instances(const float *view16, const float *inst18, int n, int w, int h, uint8_t *rgba, float *depth) {
    if (w < 32 || h < 4 || w % 32 || h % 4 || (w / 32) * (h / 4) > 128) return MV_ERR_ARG;
    // exact shading, no segmentation, a small triangle list on purpose (scenes of a few hundred triangles exercise the multi-batch path),
    // two bands when the tile rows split evenly
    const int opts[4] = {0, 0, 96, (h / 4) % 2 == 0 ? 2 : 1};
    return mv_debug_render_instances_ex(view16, inst18, n, w, h, opts, rgba, depth, nullptr, nullptr);
}

int mv_debug_cast_rays(const float *views16, const float *inst18, const int32_t *tags, const int32_t *counts, int E, int A, int stride,
                       const float *dirs3, int R, float max_dist, const uint8_t *env_mask, float *dist, uint16_t *tag) {
    if (!views16 || !inst18 || !tags || !counts || !dirs3 || !dist || !tag) return MV_ERR_ARG;
    if (E < 1 || E > 65536 || A < 1 || A > MV_MAX_AGENTS || R < 1 || R > MV_MAX_RAYS || stride < 1 || stride > 65536) return MV_ERR_ARG;
    if (size_t(E) * size_t(stride) > (size_t(1) << 22) || !std::isfinite(max_dist) || !(max_dist > 0.0f)) return MV_ERR_ARG;
    // the engine's layouts: rows [E][stride] (the entries below the env's count are cast, the rest are not read), counts [E][8] with the
    // number drawn in [1]
    std::vector<MvInstance> inst(size_t(E) * size_t(stride));
    std::vector<int32_t> cnt(size_t(E) * 8, 0);
    for (int e = 0; e < E; ++e) {
        if (counts[e] < 0 || counts[e] > stride) return MV_ERR_ARG;
        cnt[size_t(e) * 8 + 1] = counts[e];
        for (int i = 0; i < counts[e]; ++i) {
            const size_t r = size_t(e) * size_t(stride) + size_t(i);
            const float mesh = inst18[r * 18];
            if (!(mesh >= 0.0f && mesh <= 4.0f) || mesh != std::floor(mesh)) return MV_ERR_ARG;
            MvInstance &d = inst[r];
            d.mesh = int(mesh); d.color = 0;
            std::memcpy(d.model, inst18 + r * 18 + 2, 64);
            d.pad[0] = tags[r]; d.pad[1] = 0;
        }
    }
    const size_t nv = size_t(E) * size_t(A), nr = nv * size_t(R);
    DevBuf<MvInstance> dInst; DevBuf<int32_t> dCnt; DevBuf<float> dViews, dDirs, dDist; DevBuf<uint8_t> dMask; DevBuf<uint16_t> dTag;
    bool ok = dInst.alloc(inst.size()) == cudaSuccess && dCnt.alloc(cnt.size()) == cudaSuccess && dViews.alloc(nv * 16) == cudaSuccess &&
              dDirs.alloc(size_t(R) * 3) == cudaSuccess && dDist.alloc(nr) == cudaSuccess && dTag.alloc(nr) == cudaSuccess &&
              (!env_mask || dMask.alloc(size_t(E)) == cudaSuccess);
    ok = ok && cudaMemcpy(dInst.p, inst.data(), sizeof(MvInstance) * inst.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dCnt.p, cnt.data(), sizeof(int32_t) * cnt.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dViews.p, views16, nv * 64, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dDirs.p, dirs3, size_t(R) * 12, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dDist.p, dist, nr * 4, cudaMemcpyHostToDevice) == cudaSuccess && cudaMemcpy(dTag.p, tag, nr * 2, cudaMemcpyHostToDevice) == cudaSuccess &&
         (!env_mask || cudaMemcpy(dMask.p, env_mask, size_t(E), cudaMemcpyHostToDevice) == cudaSuccess);
    if (ok) {
        // the engine's launch (Engine::castRays), on the legacy stream
        mvray::RayParams rp;
        rp.instances = dInst.p; rp.instCounts = dCnt.p; rp.views = dViews.p; rp.dirs = dDirs.p; rp.envMask = dMask.p;
        rp.dist = dDist.p; rp.tag = dTag.p; rp.instStride = stride; rp.E = E; rp.A = A; rp.R = R; rp.maxDist = max_dist;
        ok = mvray::castRays(rp, nullptr) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess &&
             cudaMemcpy(dist, dDist.p, nr * 4, cudaMemcpyDeviceToHost) == cudaSuccess && cudaMemcpy(tag, dTag.p, nr * 2, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    return ok ? MV_OK : MV_ERR_CUDA;
}

int mv_debug_kcc(const int32_t *hdr8, const float *boxes10, const float *agents3, const float *query20, int n, int32_t *out_i8, float *out_f16) {
    if (!hdr8 || !boxes10 || !agents3 || !query20 || !out_i8 || !out_f16 || n < 1 || n > 65536) return MV_ERR_ARG;
    std::vector<MvBox> statics(size_t(n) * MV_MAX_OBJECTS);
    std::vector<float> rot(size_t(n) * MV_MAX_OBJECTS * 2, 0.0f);
    std::vector<MvObject> objects(size_t(n) * MV_MAX_OBJECTS);
    std::memset(statics.data(), 0, statics.size() * sizeof(MvBox));
    std::memset(objects.data(), 0, objects.size() * sizeof(MvObject));
    auto finite = [](const float *p, int k) { for (int j = 0; j < k; ++j) if (!std::isfinite(p[j])) return false; return true; };
    auto flag = [](float v) { return v == 0.0f || v == 1.0f; };
    for (int c = 0; c < n; ++c) {
        const int32_t *hd = hdr8 + size_t(c) * 8;
        const int nsPre = hd[0], ns = hd[1], no = hd[2], A = hd[3], mode = hd[4], agent = hd[5];
        if (ns < 0 || ns > MV_MAX_OBJECTS || nsPre < 0 || nsPre > ns || no < 0 || no > MV_MAX_OBJECTS || A < 1 || A > MV_MAX_AGENTS) return MV_ERR_ARG;
        if (mode < mvk::kKccSweep || mode > mvk::kKccStep || agent < 0 || agent >= A) return MV_ERR_ARG;
        const float *q = query20 + size_t(c) * 20;
        const int nq = mode == mvk::kKccSweep ? 10 : mode == mvk::kKccRecover ? 3 : 17;
        if (!finite(q, nq) || !finite(agents3 + size_t(c) * MV_MAX_AGENTS * 3, A * 3)) return MV_ERR_ARG;
        if (mode == mvk::kKccStep && (!flag(q[13]) || !flag(q[14]) || !(q[15] > 0.0f))) return MV_ERR_ARG;
        for (int j = 0; j < ns + no; ++j) {
            const bool isStatic = j < ns;
            const float *b = boxes10 + (size_t(c) * 2 * MV_MAX_OBJECTS + (isStatic ? j : MV_MAX_OBJECTS + j - ns)) * 10;
            if (!finite(b, 10) || !flag(b[6]) || !flag(b[7]) || b[3] < 0.0f || b[4] < 0.0f || b[5] < 0.0f) return MV_ERR_ARG;
            if (isStatic) {
                MvBox &d = statics[size_t(c) * MV_MAX_OBJECTS + j];
                std::memcpy(d.c, b, 12); std::memcpy(d.h, b + 3, 12);
                d.flags = (b[6] != 0.0f ? MV_SOLID : 0) | (b[7] != 0.0f ? MV_ROTATED : 0);
                rot[(size_t(c) * MV_MAX_OBJECTS + j) * 2] = b[8]; rot[(size_t(c) * MV_MAX_OBJECTS + j) * 2 + 1] = b[9];
            } else {
                if (b[7] != 0.0f) return MV_ERR_ARG;  // objects are axis-aligned
                MvObject &d = objects[size_t(c) * MV_MAX_OBJECTS + j - ns];
                std::memcpy(d.col_c, b, 12); std::memcpy(d.col_h, b + 3, 12);
                d.enabled = b[6] != 0.0f;
            }
        }
    }
    DevBuf<int32_t> dHdr, dOutI; DevBuf<MvBox> dStatics; DevBuf<MvObject> dObjects; DevBuf<float> dRot, dAgents, dQuery, dOutF;
    const size_t nA = size_t(n) * MV_MAX_AGENTS * 3;
    bool ok = dHdr.alloc(size_t(n) * 8) == cudaSuccess && dStatics.alloc(statics.size()) == cudaSuccess && dRot.alloc(rot.size()) == cudaSuccess &&
              dObjects.alloc(objects.size()) == cudaSuccess && dAgents.alloc(nA) == cudaSuccess && dQuery.alloc(size_t(n) * 20) == cudaSuccess &&
              dOutI.alloc(size_t(n) * 8) == cudaSuccess && dOutF.alloc(size_t(n) * 16) == cudaSuccess;
    ok = ok && cudaMemcpy(dHdr.p, hdr8, size_t(n) * 32, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dStatics.p, statics.data(), statics.size() * sizeof(MvBox), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dRot.p, rot.data(), rot.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dObjects.p, objects.data(), objects.size() * sizeof(MvObject), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dAgents.p, agents3, nA * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(dQuery.p, query20, size_t(n) * 80, cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        mvk::KccCaseParams kp;
        kp.hdr = dHdr.p; kp.statics = dStatics.p; kp.staticRot = dRot.p; kp.objects = dObjects.p; kp.agentPos = dAgents.p; kp.query = dQuery.p;
        kp.outI = dOutI.p; kp.outF = dOutF.p;
        const int smem = int(sizeof(mvk::WarpShared));
        ok = cudaFuncSetAttribute(mvk::kccCaseKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess;
        if (ok) mvk::kccCaseKernel<<<n, 32, smem>>>(kp);
        ok = ok && cudaGetLastError() == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess &&
             cudaMemcpy(out_i8, dOutI.p, size_t(n) * 32, cudaMemcpyDeviceToHost) == cudaSuccess &&
             cudaMemcpy(out_f16, dOutF.p, size_t(n) * 64, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    return ok ? MV_OK : MV_ERR_CUDA;
}

// host-only (no CUDA): run the product's level generator for env stream `env_seed` and dump episode `episode`'s level in
// the mv_debug_get_level layout.  Lets the CPU test-suite compare level generation with the oracle without a GPU.
static int generateHostLevel(mv::LevelOut &lo, const char *scenario, int num_agents, int env_seed, int episode, const char *const *keys,
                             const float *vals, int nparams) {
    const int sc = scenario ? mv::scenarioFromName(scenario) : -1;
    if (sc < 0 || num_agents < 1 || num_agents > MV_MAX_AGENTS || episode < 0) return MV_ERR_ARG;
    mv::FloatParams params = mv::defaultFloatParams(scenario);
    for (int i = 0; i < nparams; ++i) params[keys[i]] = vals[i];
    mv::LevelGenerator gen(scenario, num_agents, params);
    gen.seed((unsigned long)env_seed);
    try {
        for (int ep = 0; ep <= episode; ++ep) gen.generate(lo, ep, 1 << 30);
    } catch (const std::exception &ex) { g_createError = ex.what(); return MV_ERR_CAPACITY; }  // mv_last_error(NULL) tells why
    return MV_OK;
}

int mv_debug_generate_level(const char *scenario, int num_agents, int env_seed, int episode, const char *const *keys, const float *vals, int nparams,
                            int32_t *out, int cap) {
    mv::LevelOut lo;
    const int rc = generateHostLevel(lo, scenario, num_agents, env_seed, episode, keys, vals, nparams);
    if (rc != MV_OK) return rc;
    // with the spawn yaw basis bits, so the float side of spawnAgents is pinned too
    return dumpLevel(lo.level, lo.statics.data(), lo.staticRot.data(), num_agents, true, out, cap);
}

int mv_debug_grid_box(const char *scenario, int num_agents, int env_seed, int episode, const char *const *keys, const float *vals, int nparams,
                      int32_t *out6) {
    if (!out6) return MV_ERR_ARG;
    mv::LevelOut lo;
    const int rc = generateHostLevel(lo, scenario, num_agents, env_seed, episode, keys, vals, nparams);
    if (rc != MV_OK) return rc;
    for (int a = 0; a < 3; ++a) { out6[a] = lo.level.grid_org[a]; out6[3 + a] = lo.level.grid_dim[a]; }
    return MV_OK;
}

int mv_debug_bzset(const int32_t *ops, int nops, int32_t *out_xyz, int cap) {
    MvEnvState s;
    std::memset(&s, 0, sizeof s);
    mvBzInit(s);
    for (int i = 0; i < nops; ++i) {
        const int32_t *o = ops + i * 4;
        if (o[0] == 0) mvBzInsert(s, o[1], o[2], o[3]);
        else if (o[0] == 1) mvBzErase(s, o[1], o[2], o[3]);
        else mvBzClear(s);
    }
    if (s.bz_count * 3 > cap) return -s.bz_count;
    for (int i = 0; i < s.bz_count; ++i) for (int a = 0; a < 3; ++a) out_xyz[i * 3 + a] = s.bz_items[i][a];
    return s.bz_count;
}

}  // extern "C"
