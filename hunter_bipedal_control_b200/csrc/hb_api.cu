// libhunter_b200.so -- C ABI (include/hunter_b200.h) over the sm_90a kernels. Host side: context, scratch, launches, staging; the kernels
// live in the topic headers below, and this file is the library's single translation unit.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>

#include "../../include/hunter_b200.h"
#include "hb_common.cuh"
#include "hb_mpc.cuh"
#include "hb_planner.h"
#include <algorithm>
#include <climits>
#include <string>
#include <utility>
#include <atomic>
#include <mutex>
#include <cstring>
#include <thread>
#include <vector>
#include "hb_qp.cuh"
#include "hb_rbd.cuh"
#include "hb_sqp.cuh"
#include "hb_wbc.cuh"
#include "hb_hoqp.cuh"
#include "hb_rollout.cuh"
#include "hb_estimator.cuh"
#include "hb_trajectory.cuh"
#include "hb_reference.cuh"

using namespace hb;

// ---------------------------------------------------------------------------------------------- context
// A per-robot setting of the context's episodes: the first n instances have one. The device copy is allocated at max_batch by the first
// call that sets it; host keeps the validated array the copy reads.
template <class T> struct InstanceSetting {
  T* dev;
  int n;
  std::vector<T> host;
  // what the kernels of a call whose instances start at `base` (ctx->base in a chunk) read: the records from base on; unset, none
  InstanceView<T> view(int base = 0) const { return n > base ? InstanceView<T>{dev + base, n - base} : InstanceView<T>{}; }
};

struct hb_ctx {
  hb_config cfg;
  hb_wbc_settings wbc;       // WBC gains / limits / weights in force (task.info values by default; hb_wbc_set_settings, hb_load_task_info)
  int32_t wbc_form;          // the controller's WBC (HB_WBC_WEIGHTED, HB_WBC_HIERARCHICAL; hb_wbc_set_formulation)
  int device;
  cudaStream_t stream;
  cudaStream_t stream_main, stream_aux;   // the chunked host-pointer calls pipeline their chunks over these
  int base;                               // instance offset into the per-instance scratch (chunked calls)
  int64_t launches;
  void* scratch_mem;   // the scratch every context has (dxt ... res_stance), carved by hb_create from this one allocation
  // MPC scratch
  double *dxt, *dut, *perf;
  void* sqp_mem; double *lin, *proj, *rk;   // node records of the SQP pipeline (K0 -> K1 -> K2/K3), allocated by the first MPC solve
  int32_t* flags;
  // WBC scratch: the control step's desired state / input / mode, the fused WBC's status and iterations when the caller passes none
  double *xdes, *udes;
  int32_t *wstatus, *witers, *wmode;
  void* hoqp_mem; double* hoqp_scratch;   // hb_hoqp_solve_batch's lifted inequality rows and bounds (allocated by its first call)
  // hb_resident_cycle_batch_dev: references expanded over the horizon and, with event_nodes, the node grid they are expanded on
  double *cyc_xref, *cyc_swing, *cyc_tk;
  int32_t *cyc_mode, *cyc_nn;
  // resident primal solution (hb_resident_cycle_batch): solve time, trajectories, node modes (policy evaluation between MPC solves),
  // node times / interval counts (event-node grids; allocated on every context)
  SolutionRows res;
  int res_valid;                      // number of instances holding a previous solution
  double* res_sol; int res_sol_valid;   // last good WBC solution per instance (WeightedWbc fallback, W5)
  double* res_stance;                 // the device planner's latest stance positions (row N1)
  // hb_rollout_batch_dev's scratch, allocated at max_batch by its first call: commands, plan inputs -> planner -> cycle, the tick's WBC
  // solution / joint command / torques, the states held instances are put back to, the tick time, the tick's push wrench (B x 6)
  void* ro_mem;
  hb_rollout_command* ro_cmd; hb_plan_input* ro_in; hb_reference* ro_refs; hb_solve_info* ro_info; int32_t* ro_pstat;
  double *ro_t0, *ro_x0, *ro_feet, *ro_sol, *ro_jcmd, *ro_jtau, *ro_tau, *ro_held, *ro_tnow, *ro_wrench;
  double* ro_cforce; uint8_t* ro_cflag;   // the plant's contact forces and flags on a tick that records a contact channel
  // hb_rollout_estimated_batch_dev's own scratch (first such call, at max_batch): the tick's sensor readings, contact flags, estimated rbd
  void* re_mem;
  double *re_quat, *re_gyro, *re_acc, *re_jpos, *re_jvel, *re_rbd;
  uint8_t* re_flag;
  double* re_opos; uint8_t* re_ohas;   // the tick's odometry messages (with hb_rollout_set_odometry)
  // the per-robot settings of the episodes (hb_rollout_set_pushes / _plant_variations / _terrains), set by set_instances
  InstanceSetting<hb_push_schedule> pushes;
  InstanceSetting<hb_plant_variation> variations;
  InstanceSetting<hb_terrain> terrains;
  InstanceSetting<hb_goal_schedule> goals;
  // the goal each instance of the episodes captured (index, -1: none) and its target, allocated at max_batch by the first
  // hb_rollout_set_goals that sets schedules
  void* goal_mem;
  hb_target* goal_tg; int32_t* goal_idx;
  // the planner's explicit targets (hb_plan_set_targets), read by the planner calls outside the episodes
  InstanceSetting<hb_target> plan_targets;
  // the MPC latency of each instance of the episodes (hb_rollout_set_mpc_latencies), and the adopted policy of the MRT split
  // (hb_policy_update, the episodes' adoptions), allocated at max_batch by its first use; pol_have[i]: instance i has adopted one
  InstanceSetting<int32_t> latencies;
  void* pol_mem;
  SolutionRows pol;
  std::vector<uint8_t> pol_have;
  // the tracking camera of each instance of the estimated episodes (hb_rollout_set_odometry) and the cameras' state (history, bias),
  // allocated at max_batch by the first call that sets cameras
  InstanceSetting<hb_odometry_setting> odometry;
  void* odom_mem;
  OdomCamera* odom_cam;
  // each instance's WBC settings and joint PD gains in the episodes (hb_rollout_set_controller_settings)
  InstanceSetting<hb_controller_setting> controllers;
  // each instance's simulated hardware in the episodes: actuation delay, torque limits, sensor noise and offsets (hb_rollout_set_hardware)
  InstanceSetting<hb_hardware_setting> hardware;
  // each instance's gait templates and swing settings in every device planner path (hb_plan_set_settings)
  InstanceSetting<hb_planner_settings> plan_settings;
  // the recorded channels of the episodes (hb_rollout_set_channel): the caller's buffer, its instances and rows; B == 0: unset
  struct { void* buf; int B, rows; } channels[HB_CHANNELS];
  // the episode snapshots' staging (hb_episode_save_async / hb_episode_restore), allocated at max_batch by their first call: the rows'
  // context instances or source rows, and the headers a save writes
  void* snap_mem;
  int32_t* snap_src; int64_t* snap_head;
  // host-call staging, sized on demand by the calls that use it (grow): the device arena Staging carves, and the pinned host buffer of
  // hb_resident_cycle_batch's packed references / reference verdicts
  void* arena; size_t arena_cap;
  void* pinned; size_t pinned_cap;
  int last_cuda;
  size_t last_h2d_bytes;     // bytes of packed references uploaded by the last hb_resident_cycle_batch
  // optional per-kernel event timing (hb_profile_enable / hb_profile_read)
  int prof_on, prof_n;
  cudaEvent_t* prof_ev;   // 2 * PROF_MAX events
  int* prof_kind;
};

namespace {

enum { HB_OK = 0, HB_EINVAL = -1, HB_ECUDA = -2, HB_ENOMEM = -3, HB_ECAP = -4, HB_EPLAN = -5, HB_ECOMM = -6 };

#define CK(call)                                   \
  do {                                             \
    cudaError_t e__ = (call);                      \
    if (e__ != cudaSuccess) { if (ctx) ctx->last_cuda = (int)e__; return HB_ECUDA; } \
  } while (0)

constexpr int PROF_MAX = 4096;
enum { K_UNPROFILED = -1, K_BACKWARD = 0, K_FORWARD_LS = 1, K_WBC_ASSEMBLE = 2, K_QP = 3, K_OTHER = 4, K_LIN = 5, K_LQ = 6, K_NKINDS = 7 };

template <class T> cudaError_t dalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)); }

inline void prof_begin(hb_ctx* ctx, int kind) {
  if (ctx->prof_on && ctx->prof_n < PROF_MAX) { ctx->prof_kind[ctx->prof_n] = kind; cudaEventRecord(ctx->prof_ev[2 * ctx->prof_n], ctx->stream); }
}
inline void prof_end(hb_ctx* ctx) {
  if (ctx->prof_on && ctx->prof_n < PROF_MAX) { cudaEventRecord(ctx->prof_ev[2 * ctx->prof_n + 1], ctx->stream); ctx->prof_n++; }
}

// One kernel launch on ctx->stream: counted (hb_launch_count), timed under `kind` when profiling is on (K_UNPROFILED: never), launch
// error checked.
template <class... P, class... A>
int launch(hb_ctx* ctx, int kind, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  if (kind != K_UNPROFILED) prof_begin(ctx, kind);
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<A>(args)...);
  if (kind != K_UNPROFILED) prof_end(ctx);
  ctx->launches++;
  CK(cudaGetLastError());
  return HB_OK;
}

int set_device(hb_ctx* ctx) { return cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : HB_ECUDA; }

// The checks an entry point that takes (ctx, B) opens with, in this order: the context, B >= 0 and `args` (its required pointers and the
// scalars it checks up front) -> HB_EINVAL; an empty batch -> EMPTY; with CAPPED, instances beyond the context's capacity -> HB_ECAP;
// host_ok() (host data the call reads, the resident solution it needs) -> HB_EINVAL; then the switch to the context's device. The
// capacity test counts ctx->base: 0 outside a chunked call, and inside one the offset of the chunk's instances in the per-instance scratch.
enum Cap : bool { UNCAPPED = false, CAPPED = true };
constexpr int EMPTY = 1;
inline bool no_host_check() { return true; }
template <class F = bool (*)()> int enter(hb_ctx* ctx, int B, bool args, Cap cap, const F& host_ok = no_host_check) {
  if (!ctx || B < 0 || !args) return HB_EINVAL;
  if (B == 0) return EMPTY;
  if (cap && ctx->base + B > ctx->cfg.max_batch) return HB_ECAP;
  if (!host_ok()) return HB_EINVAL;
  return set_device(ctx);
}
// returns from the entry point unless enter() passed, with HB_OK for an empty batch (EMPTY never crosses the ABI)
#define ENTER(...)                                                   \
  do {                                                               \
    const int rc__ = enter(__VA_ARGS__);                             \
    if (rc__) return rc__ == EMPTY ? HB_OK : rc__;                   \
  } while (0)

// true when every one of the B records passes ok (a null array holds none); otherwise false, with the index of the first that fails in *bad
template <class T> bool all_ok(int B, const T* src, bool (*ok)(const T&), int32_t* bad = nullptr) {
  if (src) for (int i = 0; i < B; ++i) if (!ok(src[i])) { if (bad) *bad = i; return false; }
  return true;
}
// The body of hb_check_setting_records for the records of one type, judged by the predicate their setter passes to set_instances
template <class T> int check_records(int B, const void* records, bool (*ok)(const T&), int32_t* first_bad) {
  return all_ok(B, static_cast<const T*>(records), ok, first_bad) ? HB_OK : HB_EINVAL;
}

// The body of the per-robot setting calls (hunter_b200.h, "per-robot episode settings"): the records are validated on the host, B == 0
// clears the setting, a rejected call keeps the previous one and enqueues nothing, the copy goes in stream order on the context's stream.
template <class T> int set_instances(hb_ctx* ctx, int B, const T* src, bool (*ok)(const T&), InstanceSetting<T> hb_ctx::*setting) {
  const int rc = enter(ctx, B, B == 0 || src, CAPPED, [&] { return all_ok(B, src, ok); });
  if (rc == EMPTY) { (ctx->*setting).n = 0; return HB_OK; }
  if (rc) return rc;
  InstanceSetting<T>& s = ctx->*setting;
  if (!s.dev && dalloc(&s.dev, (size_t)ctx->cfg.max_batch) != cudaSuccess) { cudaGetLastError(); s.dev = nullptr; return HB_ENOMEM; }
  // a pageable copy the context owns: cudaMemcpyAsync has consumed it when it returns, whatever memory the caller's array is in
  try { s.host.assign(src, src + B); } catch (const std::bad_alloc&) { return HB_ENOMEM; }
  CK(cudaMemcpyAsync(s.dev, s.host.data(), sizeof(T) * B, cudaMemcpyHostToDevice, ctx->stream));
  s.n = B;
  return HB_OK;
}

// The validity of each kind of scalar parameter, shared by every entry point that takes it (NaN fails every test)
bool sim_params_ok(const hb_sim_params& p) { return p.dt > 0.0 && p.substeps >= 1 && p.substeps <= 1000; }
bool delay_ok(double delay) { return delay >= 0.0; }
bool cutoff_ok(double cutoff_frequency, double dt) { return cutoff_frequency > 0.0 && dt > 0.0; }
bool qp_shape_ok(int n, int m) { return n >= 1 && n <= QP_MAX_N && m >= 0 && m <= QP_MAX_M; }
bool sensor_noise_ok(const hb_sensor_noise& n) {
  for (double s : {n.orientation, n.angular_velocity, n.linear_acceleration, n.joint_position, n.joint_velocity})
    if (!(s >= 0.0) || !isfinite(s)) return false;
  return true;
}

// Waits for both streams of the context and returns rc, or the first failed wait when rc is HB_OK. Every host-pointer call ends here
// once it has queued a copy, on every exit: no copy is left reading or writing the caller's buffers, or the arena the next call may free.
int drain(hb_ctx* ctx, int rc) {
  const cudaError_t e1 = cudaStreamSynchronize(ctx->stream_aux), e0 = cudaStreamSynchronize(ctx->stream_main);
  if (rc) return rc;
  if (e0 != cudaSuccess || e1 != cudaSuccess) { ctx->last_cuda = (int)(e0 != cudaSuccess ? e0 : e1); return HB_ECUDA; }
  return HB_OK;
}

// The growth policy of the context's on-demand buffers (the staging arena, the pinned host buffer): grow only, to 5/4 of the request so
// that a packed reference stream a little longer than the last one does not reallocate, contents not kept. Every host-pointer call waits
// for its copies before it returns, so no copy still reads the buffer that is freed.
int grow(hb_ctx* ctx, void** buf, size_t* cap, size_t bytes, bool pinned_host) {
  if (bytes <= *cap) return HB_OK;
  if (*buf) { if (pinned_host) cudaFreeHost(*buf); else cudaFree(*buf); }
  *buf = nullptr; *cap = 0;
  const size_t want = bytes + bytes / 4;
  const cudaError_t e = pinned_host ? cudaHostAlloc(buf, want, cudaHostAllocDefault) : cudaMalloc(buf, want);
  if (e != cudaSuccess) { *buf = nullptr; ctx->last_cuda = (int)e; cudaGetLastError(); return HB_ENOMEM; }
  *cap = want;
  return HB_OK;
}

// Slices of one buffer, each on a 256-byte boundary as separate cudaMalloc's would place it (TMA reads need 16-byte aligned sources):
// returns the slice of n elements at byte offset `off` of base and moves `off` past it. With a null base it only measures.
template <class T> T* carve(void* base, size_t& off, size_t n) {
  T* p = base ? reinterpret_cast<T*>(static_cast<char*>(base) + off) : nullptr;
  off += (n * sizeof(T) + 255) & ~(size_t)255;
  return p;
}

// Scratch of a group of entry points, allocated by the first call that needs it: one allocation *mem, which layout(base) carves and
// whose size it returns (it is called with a null base to measure, then with the allocation). A failed allocation returns HB_ENOMEM and
// leaves the group unallocated. hb_destroy frees *mem.
template <class F> int reserve_group(void** mem, F&& layout) {
  if (*mem) return HB_OK;
  if (cudaMalloc(mem, layout(nullptr)) != cudaSuccess) { cudaGetLastError(); *mem = nullptr; return HB_ENOMEM; }
  layout(*mem);
  return HB_OK;
}

// The six rows of a solution (SolutionRows) of n instances on a horizon of N intervals, carved from base as carve does
SolutionRows carve_solution(void* base, size_t& off, size_t n, size_t N) {
  SolutionRows r;
  r.t0 = carve<double>(base, off, n); r.xt = carve<double>(base, off, n * (N + 1) * NX); r.ut = carve<double>(base, off, n * N * NU);
  r.tk = carve<double>(base, off, n * (N + 1)); r.mode = carve<int32_t>(base, off, n * (N + 1)); r.nn = carve<int32_t>(base, off, n);
  return r;
}

// Instances [o, ...) of a solution of horizon N stored at max_batch; the grid rows are null on uniform grids (grid false)
SolutionRows rows_at(const SolutionRows& r, size_t o, size_t N, bool grid) {
  return SolutionRows{r.t0 + o, r.xt + o * (N + 1) * NX, r.ut + o * N * NU, grid ? r.tk + o * (N + 1) : nullptr, r.mode + o * (N + 1),
                      grid ? r.nn + o : nullptr};
}

// Device side of one staged argument. Converts to its device pointer once Staging::reserve has placed it (null for a null pass-through
// argument); at(i) points at instance i (element i of a buf slice).
template <class T> struct Dev {
  void* const* p;
  size_t per;
  operator T*() const { return static_cast<T*>(*p); }
  T* at(size_t i) const { return static_cast<T*>(*p) + i * per; }
};

// Instances [lo, hi) of a staged call, its chunk c
struct Chunk { int c; size_t lo, hi; int n; };

// Staging of one host-pointer call. The call declares its host arguments with their elements per instance; run() then places all of
// them in the context's device arena (grown on demand, freed by hb_destroy) before any copy is enqueued. Slices start on 256-byte
// boundaries, as separate cudaMalloc's would.
//   in / inout   copied in (inout: and back)
//   out          the device always gets a buffer; copied back only when the caller passed a host pointer
//   *_or_null    a null host pointer stays a null device pointer
//   tmp / buf    device only: per instance (tmp) or n elements for the whole call (buf)
class Staging {
 public:
  Staging(hb_ctx* ctx, int B) : ctx_(ctx), B_((size_t)B) {}
  template <class T> Dev<const T> in(const T* h, size_t per) { return add<const T>(h, nullptr, per, B_, true); }
  template <class T> Dev<T> inout(T* h, size_t per) { return add<T>(h, h, per, B_, true); }
  template <class T> Dev<T> out(T* h, size_t per) { return add<T>(nullptr, h, per, B_, true); }
  template <class T> Dev<const T> in_or_null(const T* h, size_t per) { return add<const T>(h, nullptr, per, B_, h != nullptr); }
  template <class T> Dev<T> inout_or_null(T* h, size_t per) { return add<T>(h, h, per, B_, h != nullptr); }
  template <class T> Dev<T> tmp(size_t per) { return add<T>(nullptr, nullptr, per, B_, true); }
  template <class T> Dev<T> buf(size_t n) { Dev<T> d = add<T>(nullptr, nullptr, n, 1, true); d.per = 1; return d; }

  // Places the arguments, then runs the call in nchunk chunks: chunk c covers instances [B c / nchunk, B (c + 1) / nchunk) on
  // stream_main (even c) or stream_aux (odd c), so the copies of one chunk overlap the kernels of the other. Per chunk: copy in, body(k)
  // with ctx->stream / ctx->base pointing at the chunk, copy out. The first error ends the loop; ctx->stream / ctx->base are restored and
  // both streams drained before it is returned. One chunk is the whole batch on stream_main.
  template <class F> int run(int nchunk, F&& body) {
    int rc = grow(ctx_, &ctx_->arena, &ctx_->arena_cap, place(nullptr), false);
    if (rc) return rc;
    place(ctx_->arena);
    for (int c = 0; c < nchunk && rc == HB_OK; ++c) {
      const size_t lo = B_ * c / nchunk, hi = B_ * (c + 1) / nchunk;
      ctx_->stream = (c % 2 == 0) ? ctx_->stream_main : ctx_->stream_aux;
      ctx_->base = (int)lo;
      rc = copy(lo, hi, true);
      if (!rc) rc = body(Chunk{c, lo, hi, (int)(hi - lo)});
      if (!rc) rc = copy(lo, hi, false);
    }
    ctx_->stream = ctx_->stream_main;
    ctx_->base = 0;
    return drain(ctx_, rc);
  }

 private:
  struct Slot { const void* src; void* dst; size_t bytes, count; void* dev; bool used; };
  template <class T> Dev<T> add(const void* src, void* dst, size_t per, size_t count, bool used) {
    Slot& s = s_[n_++];
    s = Slot{src, dst, per * sizeof(T), count, nullptr, used};
    return Dev<T>{&s.dev, per};
  }
  // carves the used slots from base (null: measures only); returns the bytes they take
  size_t place(void* base) {
    size_t off = 0;
    for (int k = 0; k < n_; ++k) if (s_[k].used) s_[k].dev = carve<char>(base, off, s_[k].bytes * s_[k].count);
    return off;
  }
  int copy(size_t lo, size_t hi, bool to_dev) {
    hb_ctx* ctx = ctx_;
    for (int k = 0; k < n_; ++k) {
      const Slot& s = s_[k];
      const size_t off = lo * s.bytes, n = (hi - lo) * s.bytes;
      if (to_dev && s.src) CK(cudaMemcpyAsync(static_cast<char*>(s.dev) + off, static_cast<const char*>(s.src) + off, n, cudaMemcpyHostToDevice, ctx->stream));
      if (!to_dev && s.dst) CK(cudaMemcpyAsync(static_cast<char*>(s.dst) + off, static_cast<char*>(s.dev) + off, n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    return HB_OK;
  }
  hb_ctx* ctx_;
  size_t B_;
  Slot s_[16];   // the largest call (hb_resident_plan_cycle_batch) declares 11
  int n_ = 0;
};

// chunk count of the host-pointer cycles: cfg.e2e_chunks when set (one chunk below 64 instances per chunk), otherwise two from 4096
// instances on when the call has host work and copies to hide behind the other chunk's kernels (`overlap`)
int cycle_chunks(const hb_ctx* ctx, int B, bool overlap) {
  const int c = ctx->cfg.e2e_chunks;
  return c > 0 ? (B >= 64 * c ? c : 1) : ((overlap && B >= 4096) ? 2 : 1);
}

}  // namespace

extern "C" {

int hb_default_config(hb_config* cfg) {
  if (!cfg) return HB_EINVAL;
  cfg->horizon_N = 100;
  cfg->dt = 0.01;
  cfg->max_batch = 1024;
  cfg->wbc_rho = 1e-8;      // Tikhonov weight of the WBC QP: its optimum is the least-norm one to O(rho) (DESIGN.md section 2, item 4)
  cfg->qp_max_iter = 40;
  cfg->line_search_max_trials = 14;
  cfg->time_horizon = 0.0;
  cfg->event_nodes = 0;
  cfg->e2e_chunks = 0;
  return HB_OK;
}

const char* hb_strerror(int code) {
  switch (code) {
    case HB_OK: return "ok";
    case HB_EINVAL: return "invalid argument";
    case HB_ECUDA: return "CUDA error";
    case HB_ENOMEM: return "out of memory";
    case HB_ECAP: return "batch exceeds context capacity";
    case HB_EPLAN: return "reference planner: swing phase without take-off / touch-down time, or reference capacity exceeded";
    case HB_ECOMM: return "NCCL not available or a collective failed (hb_shard_last_error)";
    default: return "unknown error";
  }
}

int hb_create(const hb_config* cfg, int device, hb_ctx** out) {
  // horizon cap: the warm shift stages one instance's previous trajectories in shared memory ((2N+1) x 22 doubles <= 227 KB); its
  // kernel is opted in once at the cap below, whatever this context's horizon
  if (!cfg || !out || cfg->horizon_N < 1 || cfg->horizon_N > HB_MAX_HORIZON || cfg->max_batch < 1 || !(cfg->dt > 0.0) || cfg->time_horizon < 0.0 ||
      cfg->line_search_max_trials < 1) return HB_EINVAL;
  hb_ctx* ctx = new (std::nothrow) hb_ctx();
  if (!ctx) return HB_ENOMEM;
  memset(ctx, 0, sizeof(*ctx));
  ctx->cfg = *cfg;
  ctx->device = device;
  hb_default_wbc_settings(&ctx->wbc);
  // every failure below goes through hb_destroy (streams and partial allocations are released there)
  if (cudaSetDevice(device) != cudaSuccess) { hb_destroy(ctx); return HB_ECUDA; }
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->stream = nullptr; hb_destroy(ctx); return HB_ECUDA; }
  ctx->stream_main = ctx->stream;
  if (cudaStreamCreateWithFlags(&ctx->stream_aux, cudaStreamNonBlocking) != cudaSuccess) { ctx->stream_aux = nullptr; hb_destroy(ctx); return HB_ECUDA; }
  // model constants
  Model* m = new Model();
  memset(m, 0, sizeof(Model));
  for (int b = 0; b < NBODY; ++b) {
    for (int i = 0; i < 3; ++i) { m->joint_xyz[3 * b + i] = HB_JOINT_XYZ[3 * b + i]; m->com[3 * b + i] = HB_BODY_COM[3 * b + i]; }
    for (int i = 0; i < 9; ++i) m->inertia[9 * b + i] = HB_BODY_INERTIA[9 * b + i];
    m->mass[b] = HB_BODY_MASS[b];
    int code = 0;
    for (int i = 0; i < 3; ++i) if (HB_JOINT_AXIS[3 * b + i] != 0.0) code = (HB_JOINT_AXIS[3 * b + i] > 0 ? 1 : -1) * (i + 1);
    m->joint_axis[b] = code;
  }
  m->total_mass = HB_TOTAL_MASS;
  for (int i = 0; i < 12; ++i) m->contact_offset[i] = HB_CONTACT_OFFSET[i];
  for (int j = 0; j < NJ; ++j) { m->joint_lower[j] = HB_JOINT_LOWER[j]; m->joint_upper[j] = HB_JOINT_UPPER[j]; m->joint_vel_limit[j] = HB_JOINT_VEL_LIMIT[j]; m->torque_limit[j] = HB_WBC_TORQUE_LIMITS[j % 5]; }
  for (int i = 0; i < NX; ++i) m->Q[i] = HB_Q_DIAG[i];
  cudaError_t e = cudaMemcpyToSymbol(c_model, m, sizeof(Model));
  if (e == cudaSuccess) {
    double* dR = nullptr;
    e = dalloc(&dR, NU * NU);
    if (e == cudaSuccess) {
      init_input_cost_kernel<<<1, 32, 0, ctx->stream>>>(dR);
      e = cudaStreamSynchronize(ctx->stream);
      if (e == cudaSuccess) e = cudaMemcpy(m->R, dR, sizeof(double) * NU * NU, cudaMemcpyDeviceToHost);
      if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_model, m, sizeof(Model));
      cudaFree(dR);
    }
  }
  if (e == cudaSuccess) {
    double tab[32 * LQ_LANE_TAB] = {};
    for (int l = 0; l < 32; ++l) {
      double* t = tab + l * LQ_LANE_TAB;
      if (l < NX) t[0] = m->Q[l];
      if (l < 12) t[1] = m->R[l * NU + l];
      if (l >= 12 && l < NU) for (int j = 0; j < NJ; ++j) t[2 + j] = m->R[l * NU + 12 + j];
      if (l < 10) { t[12] = m->joint_lower[l]; t[13] = m->joint_upper[l]; }
      else if (l < 20) { t[12] = -m->joint_vel_limit[l - 10]; t[13] = m->joint_vel_limit[l - 10]; }
    }
    e = cudaMemcpyToSymbol(g_lq_lane, tab, sizeof(tab));
  }
  delete m;
  if (e != cudaSuccess) { ctx->last_cuda = (int)e; hb_destroy(ctx); return HB_ECUDA; }
  const size_t B = cfg->max_batch, N = cfg->horizon_N;
  // the node records of the SQP pipeline (31 KB per instance and interval) are allocated by the first MPC solve: contexts that only run the
  // WBC / QP / planner / estimator entry points never pay for them
  const int rc = reserve_group(&ctx->scratch_mem, [&](void* m) {
    size_t off = 0;
    ctx->dxt = carve<double>(m, off, B * (N + 1) * NX); ctx->dut = carve<double>(m, off, B * N * NU);
    ctx->perf = carve<double>(m, off, B * 4); ctx->flags = carve<int32_t>(m, off, B);
    ctx->xdes = carve<double>(m, off, B * NX); ctx->udes = carve<double>(m, off, B * NU);
    ctx->wstatus = carve<int32_t>(m, off, B); ctx->witers = carve<int32_t>(m, off, B); ctx->wmode = carve<int32_t>(m, off, B);
    ctx->cyc_xref = carve<double>(m, off, B * (N + 1) * NX); ctx->cyc_swing = carve<double>(m, off, B * (N + 1) * 24);
    ctx->cyc_mode = carve<int32_t>(m, off, B * (N + 1)); ctx->cyc_tk = carve<double>(m, off, B * (N + 1)); ctx->cyc_nn = carve<int32_t>(m, off, B);
    ctx->res = carve_solution(m, off, B, N);
    ctx->res_sol = carve<double>(m, off, B * NWBC); ctx->res_stance = carve<double>(m, off, B * 12);
    return off;
  });
  // host-pointer calls stage through ctx->arena, which the first such call sizes: contexts driven through device pointers never pay for it
  if (rc) { hb_destroy(ctx); return rc; }
  {
    cudaError_t fe = cudaSuccess;
    auto attr = [&](const void* fn, size_t bytes) { if (fe == cudaSuccess) fe = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); };
    attr((const void*)probe_flow_map_kernel, sizeof(ProbeShared));
    attr((const void*)qp_batch_kernel, 200 * 1024);
    attr((const void*)wbc_fused_kernel, wbc_fused_doubles() * sizeof(double));
    attr((const void*)hoqp_kernel, hoqp_smem_bytes());
    attr((const void*)hwbc_fused_kernel, hwbc_fused_bytes());
    attr((const void*)lin_kernel, 4 * sizeof(LinHalf) + sizeof(ChainModel));
    attr((const void*)lq_kernel, sizeof(LqShared));
    attr((const void*)riccati_kernel, sizeof(RicShared));
    attr((const void*)forward_linesearch2_kernel, sizeof(Fw2Shared));
    // the attribute is the kernel's, for the whole process, not this context's: opt in at the horizon cap so that a later context with a
    // shorter horizon cannot lower it below what a longer one still needs (180 400 B + the 4 104 B static ptk, under the 227 KB limit)
    attr((const void*)warm_shift_kernel, sizeof(double) * ((HB_MAX_HORIZON + 1) * NX + HB_MAX_HORIZON * NU));
    // these kernels reach their blocks per SM (8 for the one-block-per-instance kernels, HB_LQ_MINB for lq_kernel) only with the full
    // shared-memory carveout; do not leave it to the driver
    for (const void* fn : {(const void*)wbc_fused_kernel, (const void*)riccati_kernel, (const void*)lq_kernel, (const void*)hwbc_fused_kernel})
      if (fe == cudaSuccess) fe = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (fe != cudaSuccess) { ctx->last_cuda = (int)fe; hb_destroy(ctx); return HB_ECUDA; }
  }
  *out = ctx;
  return HB_OK;
}

int hb_destroy(hb_ctx* ctx) {
  if (!ctx) return HB_EINVAL;
  cudaSetDevice(ctx->device);
  void* const mem[] = {ctx->scratch_mem, ctx->sqp_mem, ctx->hoqp_mem, ctx->ro_mem, ctx->re_mem, ctx->goal_mem, ctx->pol_mem, ctx->odom_mem, ctx->snap_mem, ctx->arena,
                       ctx->pushes.dev, ctx->variations.dev, ctx->terrains.dev, ctx->goals.dev, ctx->plan_targets.dev, ctx->latencies.dev,
                       ctx->odometry.dev, ctx->controllers.dev, ctx->hardware.dev, ctx->plan_settings.dev};
  for (void* p : mem) if (p) cudaFree(p);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  if (ctx->prof_ev) { for (int i = 0; i < 2 * PROF_MAX; ++i) cudaEventDestroy(ctx->prof_ev[i]); delete[] ctx->prof_ev; delete[] ctx->prof_kind; }
  if (ctx->stream_aux) cudaStreamDestroy(ctx->stream_aux);
  if (ctx->stream_main) cudaStreamDestroy(ctx->stream_main);
  else if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return HB_OK;
}

int hb_sync(hb_ctx* ctx) {
  if (!ctx) return HB_EINVAL;
  CK(cudaStreamSynchronize(ctx->stream));
  return HB_OK;
}
int hb_profile_enable(hb_ctx* ctx, int on) {
  if (!ctx) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  if (on && !ctx->prof_ev) {
    ctx->prof_ev = new (std::nothrow) cudaEvent_t[2 * PROF_MAX];
    ctx->prof_kind = new (std::nothrow) int[PROF_MAX];
    if (!ctx->prof_ev || !ctx->prof_kind) return HB_ENOMEM;
    for (int i = 0; i < 2 * PROF_MAX; ++i) CK(cudaEventCreate(&ctx->prof_ev[i]));
  }
  ctx->prof_on = on ? 1 : 0;
  ctx->prof_n = 0;
  return HB_OK;
}

int hb_profile_read(hb_ctx* ctx, double* ms_per_kind, int64_t* count_per_kind) {
  if (!ctx || !ms_per_kind || !count_per_kind) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  CK(cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < K_NKINDS; ++k) { ms_per_kind[k] = 0.0; count_per_kind[k] = 0; }
  for (int i = 0; i < ctx->prof_n; ++i) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ctx->prof_ev[2 * i], ctx->prof_ev[2 * i + 1]));
    ms_per_kind[ctx->prof_kind[i]] += ms;
    count_per_kind[ctx->prof_kind[i]]++;
  }
  ctx->prof_n = 0;
  return HB_OK;
}

const char* hb_last_cuda_error(const hb_ctx* ctx) { return ctx ? cudaGetErrorString((cudaError_t)ctx->last_cuda) : "no context"; }

int64_t hb_launch_count(const hb_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t hb_last_reference_upload_bytes(const hb_ctx* ctx) { return ctx ? (int64_t)ctx->last_h2d_bytes : 0; }
void* hb_stream(hb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// ------------------------------------------------------------------------------------------ device-pointer entry points
static int launch_qp(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                     size_t sH, size_t sA, size_t sB, const int32_t* m_per, double* x, int32_t* status, int32_t* iters) {
  if (!qp_shape_ok(n, m)) return HB_EINVAL;
  const size_t per_warp = qp_workspace_doubles(n) * sizeof(double);
  int wpb = (int)((200 * 1024) / per_warp);
  if (wpb < 1) return HB_EINVAL;
  if (wpb > 1) wpb = 1;   // one warp per CTA: the shared-memory footprint, not the thread count, bounds residency
  const int blocks = (B + wpb - 1) / wpb;
  return launch(ctx, K_QP, qp_batch_kernel, blocks, 32 * wpb, per_warp * wpb, B, n, m, H, g, A, lbA, ubA, sH, sA, sB, m_per, ctx->cfg.wbc_rho,
                ctx->cfg.qp_max_iter, x, status, iters);
}

int hb_wbc_qp_batch_dev(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                        const double* ubA, double* x, int32_t* status, int32_t* iters) {
  ENTER(ctx, B, H && g && A && lbA && ubA && x, UNCAPPED);
  return launch_qp(ctx, B, n, m, H, g, A, lbA, ubA, (size_t)n * n, (size_t)m * n, (size_t)m, nullptr, x, status, iters);
}

// The instances' controller settings as the episode kernels read them; every other call passes an empty view
using ControllerView = InstanceView<hb_controller_setting>;

// hb_wbc_solve_batch_dev, with each instance of `cs` on its own WBC settings
static int wbc_solve_impl(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                          const uint8_t* stance_mode, double* sol, int32_t* status, ControllerView cs) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && sol, CAPPED);
  return launch(ctx, K_QP, wbc_fused_kernel, B, 32, wbc_fused_doubles() * sizeof(double), B, ctx->wbc, cs, x_des, u_des, rbd, mode, stance_mode,
                ctx->cfg.wbc_rho, ctx->cfg.qp_max_iter, sol, status ? status : ctx->wstatus + ctx->base, ctx->witers + ctx->base);
}

int hb_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                           const uint8_t* stance_mode, double* sol, int32_t* status) {
  return wbc_solve_impl(ctx, B, x_des, u_des, rbd, mode, stance_mode, sol, status, ControllerView{});
}

int hb_wbc_assemble_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                              const uint8_t* stance_mode, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_rows) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && H && g && A && lbA && ubA && m_rows, UNCAPPED);
  const int wpb = 4;
  return launch(ctx, K_WBC_ASSEMBLE, wbc_assemble_kernel, (B + wpb - 1) / wpb, 32 * wpb, sizeof(WbcShared) * wpb, B, ctx->wbc, x_des, u_des, rbd, mode,
                stance_mode, H, g, A, lbA, ubA, m_rows);
}

int hb_wbc_qp_rows_batch_dev(hb_ctx* ctx, int B, int n, int m_alloc, const int32_t* m_rows, const double* H, const double* g, const double* A,
                             const double* lbA, const double* ubA, double* x, int32_t* status, int32_t* iters) {
  ENTER(ctx, B, m_rows && H && g && A && lbA && ubA && x, UNCAPPED);
  return launch_qp(ctx, B, n, m_alloc, H, g, A, lbA, ubA, (size_t)n * n, (size_t)m_alloc * n, (size_t)m_alloc, m_rows, x, status, iters);
}

static int hoqp_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->hoqp_mem, [&](void* m) {
    size_t off = 0;
    ctx->hoqp_scratch = carve<double>(m, off, Bc * HQ_SCRATCH);
    return off;
  });
}

int hb_hoqp_solve_batch_dev(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack, int32_t* status) {
  ENTER(ctx, B, problems && x, CAPPED);
  const int rc = hoqp_reserve(ctx);
  if (rc) return rc;
  return launch(ctx, K_QP, hoqp_kernel, B, 32, hoqp_smem_bytes(), B, problems, ctx->hoqp_scratch, 2 * ctx->cfg.qp_max_iter, x, slack, status);
}

static int hwbc_tasks_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, hb_hoqp_problem* problems) {
  return launch(ctx, K_WBC_ASSEMBLE, hwbc_tasks_kernel, B, 32, 0, B, ctx->wbc, x_des, u_des, rbd, mode, problems);
}

// hb_hierarchical_wbc_solve_batch_dev, with each instance of `cs` on its own WBC settings
static int hwbc_solve_impl(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                           int32_t* status, ControllerView cs) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && sol, CAPPED);
  return launch(ctx, K_QP, hwbc_fused_kernel, B, 32, hwbc_fused_bytes(), B, ctx->wbc, cs, x_des, u_des, rbd, mode, 2 * ctx->cfg.qp_max_iter, sol,
                status);
}

int hb_hierarchical_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                                        int32_t* status) {
  return hwbc_solve_impl(ctx, B, x_des, u_des, rbd, mode, sol, status, ControllerView{});
}

// The controller's WBC (LeggedController::wbc_) on device pointers: every entry point that runs it comes through here. stance_mode is read
// by the weighted formulation only (WbcBase::setStanceMode reaches only WeightedWbc::formulateWeightedTasks). status: nullable, as for
// hb_wbc_solve_batch_dev. cs: the episodes' controller settings, empty for every other caller.
static int controller_wbc_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                              const uint8_t* stance_mode, double* sol, int32_t* status, ControllerView cs = ControllerView{}) {
  if (ctx->wbc_form == HB_WBC_HIERARCHICAL)
    return hwbc_solve_impl(ctx, B, x_des, u_des, rbd, mode, sol, status ? status : ctx->wstatus + ctx->base, cs);
  return wbc_solve_impl(ctx, B, x_des, u_des, rbd, mode, stance_mode, sol, status, cs);
}

int hb_mpc_cold_start_batch_dev(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj) {
  ENTER(ctx, B, x0 && mode && x_traj && u_traj, UNCAPPED);
  return launch(ctx, K_UNPROFILED, cold_start_kernel, B, 128, 0, B, ctx->cfg.horizon_N, x0, mode, x_traj, u_traj);
}

static int mpc_solve_impl(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                          double* x_traj, double* u_traj, hb_solve_info* info, const double* tk, const int32_t* nn) {
  ENTER(ctx, B, x0 && x_ref && swing_ref && mode && x_traj && u_traj && (tk == nullptr) == (nn == nullptr), CAPPED);
  const size_t Bc = ctx->cfg.max_batch, Nc = ctx->cfg.horizon_N;
  int rc = reserve_group(&ctx->sqp_mem, [&](void* m) {
    size_t off = 0;
    ctx->lin = carve<double>(m, off, Bc * Nc * LIN_STRIDE); ctx->proj = carve<double>(m, off, Bc * Nc * PJ_STRIDE);
    ctx->rk = carve<double>(m, off, Bc * Nc * RK_STRIDE);
    return off;
  });
  if (rc) return rc;
  SqpArgs a;
  a.tk = tk; a.nn = nn;
  a.B = B; a.N = ctx->cfg.horizon_N; a.dt = ctx->cfg.dt; a.x_ref = x_ref; a.swing = swing_ref; a.mode = mode; a.xt = x_traj; a.ut = u_traj;
  {
    const size_t o = (size_t)ctx->base, Nn = (size_t)ctx->cfg.horizon_N;
    a.lin = ctx->lin + o * Nn * LIN_STRIDE; a.proj = ctx->proj + o * Nn * PJ_STRIDE; a.rk = ctx->rk + o * Nn * RK_STRIDE;
    a.dxt = ctx->dxt + o * (Nn + 1) * NX; a.dut = ctx->dut + o * Nn * NU; a.perf = ctx->perf + o * 4; a.flags = ctx->flags + o; a.x0 = x0;
  }
  const int N = a.N, NP = (N + 1) / 2;
  const long long nw = (long long)B * NP;
  rc = launch(ctx, K_LIN, lin_kernel, (unsigned)((nw + 1) / 2), 64, 4 * sizeof(LinHalf) + sizeof(ChainModel), a);
  if (!rc) rc = launch(ctx, K_LQ, lq_kernel, (unsigned)((long long)B * N), 32, sizeof(LqShared), a);
  if (!rc) rc = launch(ctx, K_BACKWARD, riccati_kernel, B, 64, sizeof(RicShared), a);
  if (!rc) rc = launch(ctx, K_FORWARD_LS, forward_linesearch2_kernel, B, 32, sizeof(Fw2Shared), a, ctx->cfg.line_search_max_trials, info);
  return rc;
}

int hb_mpc_solve_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                           double* x_traj, double* u_traj, hb_solve_info* info) {
  return mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, nullptr, nullptr);
}

int hb_mpc_solve_grid_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                                const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info) {
  if (!node_times || !n_intervals) return HB_EINVAL;
  return mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, node_times, n_intervals);
}

static int policy_eval_impl(hb_ctx* ctx, int B, double t_rel, const double* x_traj, const double* u_traj, const int32_t* mode, double* x_des,
                            double* u_des, int32_t* mode_out, const double* tk, const int32_t* nn) {
  ENTER(ctx, B, x_traj && u_traj && mode && x_des && u_des && (tk == nullptr) == (nn == nullptr), UNCAPPED);
  // the caller's solution, which the kernel only reads; no solve time: it is evaluated at t_rel
  const SolutionRows s{nullptr, const_cast<double*>(x_traj), const_cast<double*>(u_traj), const_cast<double*>(tk), const_cast<int32_t*>(mode),
                       const_cast<int32_t*>(nn)};
  const int wpb = 4;
  return launch(ctx, K_UNPROFILED, policy_eval_kernel, (B + wpb - 1) / wpb, 32 * wpb, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, t_rel, s, x_des, u_des,
                mode_out, nullptr, PolicyChoice{});
}

int hb_policy_eval_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x_traj, const double* u_traj, const int32_t* mode, double* x_des,
                             double* u_des, int32_t* mode_out) {
  return policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, x_des, u_des, mode_out, nullptr, nullptr);
}

int hb_policy_eval_grid_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* node_times, const int32_t* n_intervals, const double* x_traj,
                                  const double* u_traj, const int32_t* mode, double* x_des, double* u_des, int32_t* mode_out) {
  if (!node_times || !n_intervals) return HB_EINVAL;
  return policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, x_des, u_des, mode_out, node_times, n_intervals);
}

int hb_time_grid_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals, int32_t* status) {
  ENTER(ctx, B, t0 && refs && node_times && n_intervals, UNCAPPED);
  const double T = ctx->cfg.time_horizon > 0.0 ? ctx->cfg.time_horizon : ctx->cfg.horizon_N * ctx->cfg.dt;
  return launch(ctx, K_UNPROFILED, time_grid_kernel, (B + 127) / 128, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, T, t0, refs, node_times, n_intervals, status);
}

static int control_step_impl(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                             const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                             int32_t* wbc_status, const double* tk, const int32_t* nn) {
  ENTER(ctx, B, x0 && x_ref && swing_ref && mode && rbd && x_traj && u_traj && wbc_sol && (tk == nullptr) == (nn == nullptr), CAPPED);
  int rc = mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, tk, nn);
  if (rc) return rc;
  double* xdes = ctx->xdes + (size_t)ctx->base * NX; double* udes = ctx->udes + (size_t)ctx->base * NU; int32_t* wmode = ctx->wmode + ctx->base;
  rc = policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, xdes, udes, wmode, tk, nn);
  if (rc) return rc;
  rc = controller_wbc_dev(ctx, B, xdes, udes, rbd, wmode, nullptr, wbc_sol, wbc_status);
  if (!rc && torque) rc = launch(ctx, K_UNPROFILED, torque_kernel, (B * NJ + 127) / 128, 128, 0, B, wbc_sol, torque);
  return rc;
}

int hb_control_step_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                              const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                              int32_t* wbc_status) {
  return control_step_impl(ctx, B, t_rel, x0, x_ref, swing_ref, mode, rbd, x_traj, u_traj, info, wbc_sol, torque, wbc_status, nullptr, nullptr);
}

// The WeightedWbc fallback after a resident WBC solve (wbc_fallback_kernel), when the caller asked for its status; no_prev: there is no
// previous solution to fall back to (a cold start, or its first tick). The solved instances' solutions become the new previous ones.
static int wbc_fallback(hb_ctx* ctx, int B, bool no_prev, const int32_t* wbc_status, double* wbc_sol, double* torque) {
  if (!wbc_status) return HB_OK;
  const int have_prev = (!no_prev && ctx->res_sol_valid >= ctx->base + B) ? 1 : 0;
  const int rc = launch(ctx, K_UNPROFILED, wbc_fallback_kernel, (B * NWBC + 127) / 128, 128, 0, B, have_prev, wbc_status, wbc_sol,
                        ctx->res_sol + (size_t)ctx->base * NWBC, torque);
  if (rc) return rc;
  if (ctx->res_sol_valid < ctx->base + B) ctx->res_sol_valid = ctx->base + B;
  return HB_OK;
}

// hb_resident_cycle_batch_dev; with run_wbc = false the cycle ends after the SQP iteration (hb_rollout_batch_dev: the 500 Hz tick at the
// same time is the WBC of that cycle, so the cycle's own would be thrown away)
static int resident_cycle_impl(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                               const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status, bool run_wbc) {
  ENTER(ctx, B, t0 && x0 && refs && rbd, CAPPED, [&] { return cold_start || ctx->res_valid >= ctx->base + B; });   // a warm start shifts the previous solution
  const size_t N = ctx->cfg.horizon_N, o = (size_t)ctx->base;
  double* xref = ctx->cyc_xref + o * (N + 1) * NX; double* swing = ctx->cyc_swing + o * (N + 1) * 24; int32_t* mode = ctx->cyc_mode + o * (N + 1);
  // event-node grids (cfg.event_nodes): per-instance node times, kept resident beside the primal solution
  const bool grid = ctx->cfg.event_nodes != 0;
  const SolutionRows res = rows_at(ctx->res, o, N, grid);
  double* tk = grid ? ctx->cyc_tk + o * (N + 1) : nullptr; int32_t* nn = grid ? ctx->cyc_nn + o : nullptr;
  int rc = HB_OK;
  if (grid) {
    rc = hb_time_grid_batch_dev(ctx, B, t0, refs, tk, nn, nullptr);
    if (rc) return rc;
    rc = hb_reference_expand_grid_batch_dev(ctx, B, tk, refs, xref, swing, mode);
  } else {
    rc = hb_reference_expand_batch_dev(ctx, B, t0, refs, xref, swing, mode);
  }
  if (rc) return rc;
  if (cold_start) {
    rc = hb_mpc_cold_start_batch_dev(ctx, B, x0, mode, res.xt, res.ut);
    if (!rc) rc = launch(ctx, K_UNPROFILED, set_times_kernel, (B + 127) / 128, 128, 0, B, (int)N, t0, tk, nn, res);
  } else {
    const size_t smem = sizeof(double) * ((N + 1) * NX + N * NU);     // opted in at hb_create
    rc = launch(ctx, K_UNPROFILED, warm_shift_kernel, B, 128, smem, B, (int)N, ctx->cfg.dt, t0, x0, mode, tk, nn, res);
  }
  if (rc) return rc;
  CK(cudaMemcpyAsync(res.mode, mode, sizeof(int32_t) * B * (N + 1), cudaMemcpyDeviceToDevice, ctx->stream));
  if (ctx->res_valid < ctx->base + B) ctx->res_valid = ctx->base + B;
  if (!run_wbc) return mpc_solve_impl(ctx, B, x0, xref, swing, mode, res.xt, res.ut, info, tk, nn);
  rc = control_step_impl(ctx, B, t_rel, x0, xref, swing, mode, rbd, res.xt, res.ut, info, wbc_sol, torque, wbc_status, tk, nn);
  return rc ? rc : wbc_fallback(ctx, B, cold_start != 0, wbc_status, wbc_sol, torque);
}

int hb_resident_cycle_batch_dev(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                                const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status) {
  if (!wbc_sol) return HB_EINVAL;
  return resident_cycle_impl(ctx, B, cold_start, t_rel, t0, x0, refs, rbd, info, wbc_sol, torque, wbc_status, true);
}

static const hbplan::PlanConsts& plan_consts() {
  static const hbplan::PlanConsts pc = hbplan::make_consts();
  return pc;
}

// The device planner after the entry checks: an instance with a record in targets plans on it where captured is null or captured[i] >= 0;
// an instance with a record in settings plans with it
static int plan_dev(hb_ctx* ctx, int B, const hb_plan_input* in, const double* feet, double* latest_stance, hb_reference* out, int32_t* status,
                    InstanceView<hb_target> targets, const int32_t* captured, InstanceView<hb_planner_settings> settings) {
  return launch(ctx, K_UNPROFILED, plan_references_coop_kernel, (B + 7) / 8, 32, 0, B, in, feet, latest_stance, out, status, plan_consts(), targets,
                captured, settings);
}

int hb_plan_references_batch_dev(hb_ctx* ctx, int B, const hb_plan_input* in, const double* feet, double* latest_stance, hb_reference* out,
                                 int32_t* status) {
  ENTER(ctx, B, in && latest_stance && out, UNCAPPED);
  return plan_dev(ctx, B, in, feet, latest_stance, out, status, ctx->plan_targets.view(ctx->base), nullptr, ctx->plan_settings.view(ctx->base));
}

int hb_default_kf_params(hb_kf_params* p) {
  if (!p) return HB_EINVAL;
  p->foot_radius = 0.02; p->imu_process_noise_position = 0.02; p->imu_process_noise_velocity = 0.02; p->foot_process_noise_position = 0.5;
  p->foot_sensor_noise_position = 0.5; p->foot_sensor_noise_velocity = 0.1; p->foot_height_sensor_noise = 0.01;
  return HB_OK;
}

int hb_kf_reset(int B, hb_kf_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    memset(&state[i], 0, sizeof(hb_kf_state));
    for (int k = 0; k < 18; ++k) state[i].P[k * 18 + k] = 100.0;
  }
  return HB_OK;
}

int hb_estimator_update_batch_dev(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                                  const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos, const double* joint_vel,
                                  const uint8_t* contact_flag, double* rbd_out) {
  ENTER(ctx, B, params && state && quat && ang_vel_local && lin_acc_local && joint_pos && joint_vel && contact_flag && rbd_out, UNCAPPED);
  return launch(ctx, K_UNPROFILED, kf_update_kernel<hb_kf_state, false>, B, 32, sizeof(KfShared), B, *params, dt, state, quat, ang_vel_local, lin_acc_local,
                joint_pos, joint_vel, contact_flag, rbd_out, (const double*)nullptr, (const uint8_t*)nullptr);
}

int hb_estimator_fuse_odometry_async(hb_ctx* ctx, int B, const hb_kf_params* params, hb_kf_state* state, const double* pos, const uint8_t* has_msg,
                                     const uint8_t* contact_flag, double* rbd) {
  ENTER(ctx, B, params && state && pos && has_msg && contact_flag && rbd, UNCAPPED);
  return launch(ctx, K_UNPROFILED, odometry_fuse_kernel, (B + 63) / 64, 64, 0, B, params->foot_radius, state, pos, has_msg, contact_flag, rbd);
}

int hb_default_wbc_settings(hb_wbc_settings* s) {
  if (!s) return HB_EINVAL;
  for (int j = 0; j < 5; ++j) s->torque_limits[j] = HB_WBC_TORQUE_LIMITS[j];
  s->friction_coefficient = HB_WBC_FRICTION_MU;
  s->swing_kp = HB_WBC_SWING_KP; s->swing_kd = HB_WBC_SWING_KD;
  s->base_accel_kp = 40.0; s->base_accel_kd = 4.0;            // task.info:310-314; loaded (WbcBase.cpp:386-393) but used by no task
  s->base_height_kp = HB_WBC_BASE_HEIGHT_KP; s->base_height_kd = HB_WBC_BASE_HEIGHT_KD;
  s->base_angular_kp = HB_WBC_BASE_ANGULAR_KP; s->base_angular_kd = HB_WBC_BASE_ANGULAR_KD;
  s->weight_swing_leg = HB_WBC_WEIGHT_SWING; s->weight_base_accel = HB_WBC_WEIGHT_BASE; s->weight_contact_force = HB_WBC_WEIGHT_FORCE;
  return HB_OK;
}

int hb_wbc_get_settings(const hb_ctx* ctx, hb_wbc_settings* s) {
  if (!ctx || !s) return HB_EINVAL;
  *s = ctx->wbc;
  return HB_OK;
}

int hb_wbc_set_settings(hb_ctx* ctx, const hb_wbc_settings* s) {
  if (!ctx || !s) return HB_EINVAL;
  for (int j = 0; j < 5; ++j) if (!(s->torque_limits[j] > 0.0)) return HB_EINVAL;
  if (!(s->friction_coefficient > 0.0) || !(s->weight_swing_leg > 0.0) || !(s->weight_base_accel > 0.0) || s->weight_contact_force < 0.0) return HB_EINVAL;
  ctx->wbc = *s;      // passed by value with the next launch: nothing in flight is affected
  return HB_OK;
}

int hb_wbc_set_formulation(hb_ctx* ctx, int32_t formulation) {
  if (!ctx || (formulation != HB_WBC_WEIGHTED && formulation != HB_WBC_HIERARCHICAL)) return HB_EINVAL;
  ctx->wbc_form = formulation;      // read on the host by the next launch: nothing in flight is affected
  return HB_OK;
}

int hb_wbc_get_formulation(const hb_ctx* ctx, int32_t* formulation) {
  if (!ctx || !formulation) return HB_EINVAL;
  *formulation = ctx->wbc_form;
  return HB_OK;
}

int hb_wbc_set_kp_kd(hb_ctx* ctx, double swing_kp, double swing_kd) {
  if (!ctx) return HB_EINVAL;
  ctx->wbc.swing_kp = swing_kp; ctx->wbc.swing_kd = swing_kd;
  return HB_OK;
}

namespace {
// Minimal reader of the boost property-tree INFO subset the reference's task.info uses: `key value`, `key { ... }`, `(i,j) value`,
// `;` comments. Values are collected under dotted paths ("swingLegTask.kp", "torqueLimitsTask.(0,0)").
struct InfoMap {
  std::vector<std::pair<std::string, std::string>> kv;
  const std::string* find(const std::string& k) const { for (const auto& e : kv) if (e.first == k) return &e.second; return nullptr; }
  bool number(const std::string& k, double* out) const {
    const std::string* v = find(k);
    if (!v) return false;
    char* end = nullptr;
    const double d = strtod(v->c_str(), &end);
    if (end == v->c_str()) { if (*v == "true") { *out = 1.0; return true; } if (*v == "false") { *out = 0.0; return true; } return false; }
    *out = d;
    return true;
  }
};
bool info_parse(const char* path, InfoMap& out) {
  FILE* f = fopen(path, "r");
  if (!f) return false;
  std::vector<std::string> tok;
  std::string cur;
  int ch;
  bool comment = false;
  auto flush = [&]() { if (!cur.empty()) { tok.push_back(cur); cur.clear(); } };
  while ((ch = fgetc(f)) != EOF) {
    if (comment) { if (ch == '\n') comment = false; continue; }
    if (ch == ';') { flush(); comment = true; continue; }
    if (ch == '{' || ch == '}') { flush(); tok.push_back(std::string(1, (char)ch)); continue; }
    if (ch == ' ' || ch == '\t' || ch == '\n' || ch == '\r') { flush(); continue; }
    cur.push_back((char)ch);
  }
  flush();
  fclose(f);
  std::vector<std::string> path_stack;
  size_t i = 0;
  while (i < tok.size()) {
    const std::string& t = tok[i];
    if (t == "}") { if (path_stack.empty()) return false; path_stack.pop_back(); ++i; continue; }
    if (t == "{") return false;
    if (i + 1 < tok.size() && tok[i + 1] == "{") { path_stack.push_back(t); i += 2; continue; }
    if (i + 1 >= tok.size() || tok[i + 1] == "}") { ++i; continue; }      // key without a value
    std::string key;
    for (const auto& p : path_stack) { key += p; key += '.'; }
    key += t;
    out.kv.emplace_back(key, tok[i + 1]);
    i += 2;
  }
  return path_stack.empty();
}
}  // namespace

int hb_parse_task_info(const char* path, hb_task_info* out) {
  if (!path || !out) return HB_EINVAL;
  InfoMap m;
  if (!info_parse(path, m)) return HB_EINVAL;
  memset(out, 0, sizeof(*out));
  hb_default_wbc_settings(&out->wbc);
  hb_kf_params kf; hb_default_kf_params(&kf);
  memcpy(out->kalman, &kf, sizeof(kf));
  out->contact_force_cutoff_frequency = 250.0; out->contact_threshold = 75.0;
  out->sqp_dt = 0.015; out->sqp_iteration = 1; out->mpc_time_horizon = 0.8; out->mpc_cold_start = 0;
  double v;
  int found = 0;
  hb_wbc_settings& w = out->wbc;
  for (int j = 0; j < 5; ++j) { char k[64]; snprintf(k, sizeof(k), "torqueLimitsTask.(%d,0)", j); if (m.number(k, &v)) { w.torque_limits[j] = v; found |= 1; } }
  if (m.number("frictionConeTask.frictionCoefficient", &v)) { w.friction_coefficient = v; found |= 1; }
  if (m.number("swingLegTask.kp", &v)) { w.swing_kp = v; found |= 1; }
  if (m.number("swingLegTask.kd", &v)) { w.swing_kd = v; found |= 1; }
  if (m.number("baseAccelTask.kp", &v)) { w.base_accel_kp = v; found |= 1; }
  if (m.number("baseAccelTask.kd", &v)) { w.base_accel_kd = v; found |= 1; }
  if (m.number("baseHeightTask.kp", &v)) { w.base_height_kp = v; found |= 1; }
  if (m.number("baseHeightTask.kd", &v)) { w.base_height_kd = v; found |= 1; }
  if (m.number("baseAngularTask.kp", &v)) { w.base_angular_kp = v; found |= 1; }
  if (m.number("baseAngularTask.kd", &v)) { w.base_angular_kd = v; found |= 1; }
  if (m.number("weight.swingLeg", &v)) { w.weight_swing_leg = v; found |= 1; }
  if (m.number("weight.baseAccel", &v)) { w.weight_base_accel = v; found |= 1; }
  if (m.number("weight.contactForce", &v)) { w.weight_contact_force = v; found |= 1; }
  const char* kfk[7] = {"footRadius", "imuProcessNoisePosition", "imuProcessNoiseVelocity", "footProcessNoisePosition", "footSensorNoisePosition",
                        "footSensorNoiseVelocity", "footHeightSensorNoise"};
  for (int j = 0; j < 7; ++j) if (m.number(std::string("kalmanFilter.") + kfk[j], &v)) { out->kalman[j] = v; found |= 2; }
  if (m.number("contactForceEsimation.cutoffFrequency", &v)) { out->contact_force_cutoff_frequency = v; found |= 4; }
  if (m.number("contactForceEsimation.contactThreshold", &v)) { out->contact_threshold = v; found |= 4; }
  if (m.number("sqp.dt", &v)) { out->sqp_dt = v; found |= 8; }
  if (m.number("sqp.sqpIteration", &v)) { out->sqp_iteration = (int32_t)v; found |= 8; }
  if (m.number("mpc.timeHorizon", &v)) { out->mpc_time_horizon = v; found |= 16; }
  if (m.number("mpc.coldStart", &v)) { out->mpc_cold_start = v != 0.0; found |= 16; }
  out->found = found;
  return HB_OK;
}

int hb_load_task_info(hb_ctx* ctx, const char* path) {
  if (!ctx || !path) return HB_EINVAL;
  hb_task_info ti;
  int rc = hb_parse_task_info(path, &ti);
  if (rc) return rc;
  return hb_wbc_set_settings(ctx, &ti.wbc);
}

// The ranges of hunter_b200.h's hb_planner_settings (NaN fails every test); the entries beyond n_phase are not read
static bool planner_settings_ok(const hb_planner_settings& s) {
  for (const hb_gait_template& g : s.gait) {
    if (g.n_phase < 1 || g.n_phase > HB_GAIT_MAX_PHASES || !(g.switching_times[0] == 0.0)) return false;
    for (int k = 0; k < g.n_phase; ++k) {
      if (g.modes[k] < 0 || g.modes[k] > 3) return false;
      if (!(g.switching_times[k + 1] > g.switching_times[k]) || !isfinite(g.switching_times[k + 1])) return false;
    }
  }
  if (!isfinite(s.swing_height) || !(s.swing_height >= 0.0) || !isfinite(s.swing_time_scale) || !(s.swing_time_scale > 0.0)) return false;
  for (double v : {s.next_stance_z, s.feet_bias_x1, s.feet_bias_x2, s.feet_bias_y, s.feet_bias_z}) if (!isfinite(v)) return false;
  return true;
}

int hb_default_planner_settings(hb_planner_settings* s) {
  if (!s) return HB_EINVAL;
  hbplan::default_settings(*s);
  return HB_OK;
}

namespace {
// string2ModeNumber (MotionPhaseDefinition.h:57-60, :117-125) for the biped's modes; -1 for any other name
int mode_number(const std::string& name) {
  const char* names[4] = {"FLY", "R", "L", "STANCE"};
  for (int m = 0; m < 4; ++m) if (name == names[m]) return m;
  return -1;
}
// loadModeSequenceTemplate (ModeSequenceTemplate.cpp:59-83) of the template `name`: returns 1 with *t filled, 0 when the file has neither
// of its lists, -1 when they are malformed (an unknown mode name, a non-numeric time, counts that are not n and n + 1, n > HB_GAIT_MAX_PHASES)
int gait_template_from(const InfoMap& m, const std::string& name, hb_gait_template* t) {
  memset(t, 0, sizeof(*t));
  int nm = 0, nt = 0;
  for (const std::string* v; (v = m.find(name + ".modeSequence.[" + std::to_string(nm) + "]")); ++nm) {
    if (nm == HB_GAIT_MAX_PHASES) return -1;
    if ((t->modes[nm] = mode_number(*v)) < 0) return -1;
  }
  for (std::string k; m.find(k = name + ".switchingTimes.[" + std::to_string(nt) + "]"); ++nt)
    if (nt == HB_GAIT_MAX_PHASES + 1 || !m.number(k, &t->switching_times[nt])) return -1;
  if (nm == 0 && nt == 0) return 0;
  if (nm == 0 || nt != nm + 1) return -1;
  t->n_phase = nm;
  return 1;
}
}  // namespace

int hb_parse_planner_settings(const char* task_info, const char* gait_info, hb_planner_settings* out) {
  if (!task_info || !gait_info || !out) return HB_EINVAL;
  InfoMap task, gait;
  if (!info_parse(task_info, task) || !info_parse(gait_info, gait)) return HB_EINVAL;
  hb_planner_settings s;
  hbplan::default_settings(s);
  // loadSwingTrajectorySettings (SwingTrajectoryPlanner.cpp:549-561): the fields the planner reads; an absent key keeps its default
  const std::pair<const char*, double*> swing[] = {{"swingHeight", &s.swing_height}, {"swingTimeScale", &s.swing_time_scale},
                                                   {"next_position_z", &s.next_stance_z}, {"feet_bias_x1", &s.feet_bias_x1},
                                                   {"feet_bias_x2", &s.feet_bias_x2}, {"feet_bias_y", &s.feet_bias_y}, {"feet_bias_z", &s.feet_bias_z}};
  for (const auto& f : swing) task.number(std::string("swing_trajectory_config.") + f.first, f.second);
  // gait.info: gait g is the template named by list.[g]
  for (int g = 0; g < 4; ++g) {
    const std::string* name = gait.find("list.[" + std::to_string(g) + "]");
    if (!name) continue;
    hb_gait_template t;
    const int rc = gait_template_from(gait, *name, &t);
    if (rc < 0) return HB_EINVAL;
    if (rc > 0) s.gait[g] = t;
  }
  if (!planner_settings_ok(s)) return HB_EINVAL;
  *out = s;
  return HB_OK;
}

int hb_default_sim_params(hb_sim_params* p) {
  if (!p) return HB_EINVAL;
  p->dt = 0.002; p->substeps = 4; p->ground_height = 0.0; p->ground_stiffness = 3.0e4; p->ground_damping = 3.0e2; p->tangential_damping = 3.0e2; p->friction_mu = 0.7;
  p->joint_armature = 0.1; p->joint_damping = 1.0;       // mujoco/model/hunter/hunter.xml:6 (default joint armature / damping of the reference's plant)
  return HB_OK;
}

int hb_actuation_reset(int B, hb_actuation_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  memset(state, 0, sizeof(hb_actuation_state) * (size_t)B);       // cmdBuffer_ cleared (LeggedHWSim.cpp:171-174)
  return HB_OK;
}

// The instances' simulated hardware as the actuation, saturation and sensor kernels read it; the calls without records pass an empty view
using HardwareView = InstanceView<hb_hardware_setting>;

// The ranges of hunter_b200.h's hb_hardware_setting: every field finite, delay >= 0, limits > 0, sigmas >= 0
static bool hardware_setting_ok(const hb_hardware_setting& s) {
  const double* f = reinterpret_cast<const double*>(&s);
  static_assert(sizeof(hb_hardware_setting) == 35 * sizeof(double), "hb_hardware_setting holds 35 doubles");
  for (int i = 0; i < 35; ++i) if (!isfinite(f[i])) return false;
  if (!delay_ok(s.actuation_delay)) return false;
  for (double lim : s.torque_limit) if (!(lim > 0.0)) return false;
  for (double sigma : {s.sigma_orientation, s.sigma_angular_velocity, s.sigma_linear_acceleration, s.sigma_joint_position, s.sigma_joint_velocity})
    if (!(sigma >= 0.0)) return false;
  return true;
}

int hb_default_hardware_setting(hb_hardware_setting* s) {
  if (!s) return HB_EINVAL;
  memset(s, 0, sizeof(*s));
  hb_rollout_params p;            // the delay and limits of the default episode
  hb_default_rollout_params(&p);
  s->actuation_delay = p.actuation_delay;
  for (int j = 0; j < NJ; ++j) s->torque_limit[j] = p.torque_limit[j];
  return HB_OK;
}

int hb_rollout_set_hardware(hb_ctx* ctx, int B, const hb_hardware_setting* s) { return set_instances(ctx, B, s, hardware_setting_ok, &hb_ctx::hardware); }

// hb_actuation_batch_dev, with each instance of `hw` on its own delay (the episodes, hb_actuation_hw)
static int actuation_dev(hb_ctx* ctx, int B, double delay, HardwareView hw, const double* time, hb_actuation_state* state, const double* command,
                         const double* rbd, double* tau) {
  ENTER(ctx, B, time && state && command && rbd && tau && delay_ok(delay), UNCAPPED);
  return launch(ctx, K_UNPROFILED, actuation_kernel, (B + 63) / 64, 64, 0, B, delay, hw, time, state, command, rbd, tau);
}

int hb_actuation_batch_dev(hb_ctx* ctx, int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd,
                           double* tau) {
  return actuation_dev(ctx, B, delay, HardwareView{}, time, state, command, rbd, tau);
}

// the plant step after the entry checks; wrench (B x 6) nullable; var: the plants of the instances, ter: the ground under them
static int sim_step(hb_ctx* ctx, int B, const hb_sim_params& params, double* rbd, const double* tau, const double* wrench,
                    InstanceView<hb_plant_variation> var, InstanceView<hb_terrain> ter, double* contact_force, uint8_t* contact_flag) {
  return launch(ctx, K_UNPROFILED, sim_step_kernel, B, 32, 0, B, params, rbd, tau, wrench, var, ter, contact_force, contact_flag);
}

int hb_sim_step_batch_dev(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force, uint8_t* contact_flag) {
  ENTER(ctx, B, params && rbd && tau && sim_params_ok(*params), UNCAPPED);
  return sim_step(ctx, B, *params, rbd, tau, nullptr, {}, {}, contact_force, contact_flag);
}

int hb_default_plant_variation(hb_plant_variation* v) {
  if (!v) return HB_EINVAL;
  memset(v, 0, sizeof(*v));
  v->friction_scale = 1.0; v->stiffness_scale = 1.0; v->damping_scale = 1.0;
  for (int j = 0; j < NJ; ++j) v->motor_strength[j] = 1.0;
  return HB_OK;
}

// The ranges of hunter_b200.h's hb_plant_variation. The payload inertia is checked for exact symmetry and, by Sylvester's criterion for
// semidefiniteness, for no negative principal minor (the three diagonal entries, the three 2 x 2 minors and the determinant).
static bool plant_variation_ok(const hb_plant_variation& v) {
  const double* I = v.payload_inertia;
  auto finite = [](const double* x, int n) { for (int i = 0; i < n; ++i) if (!isfinite(x[i])) return false; return true; };
  if (!finite(&v.payload_mass, 1) || !finite(v.payload_com, 3) || !finite(I, 9) || !finite(&v.friction_scale, 1) || !finite(&v.stiffness_scale, 1) ||
      !finite(&v.damping_scale, 1) || !finite(v.motor_strength, NJ))
    return false;
  if (!(v.payload_mass >= 0.0) || !(v.friction_scale >= 0.0) || !(v.stiffness_scale > 0.0) || !(v.damping_scale >= 0.0)) return false;
  for (int j = 0; j < NJ; ++j) if (!(v.motor_strength[j] >= 0.0)) return false;
  if (I[1] != I[3] || I[2] != I[6] || I[5] != I[7]) return false;
  if (I[0] < 0.0 || I[4] < 0.0 || I[8] < 0.0) return false;
  if (I[0] * I[4] - I[1] * I[3] < 0.0 || I[0] * I[8] - I[2] * I[6] < 0.0 || I[4] * I[8] - I[5] * I[7] < 0.0) return false;
  const double det = I[0] * (I[4] * I[8] - I[5] * I[7]) - I[1] * (I[3] * I[8] - I[5] * I[6]) + I[2] * (I[3] * I[7] - I[4] * I[6]);
  if (det < 0.0) return false;
  if (v.payload_mass == 0.0) {
    for (int i = 0; i < 3; ++i) if (v.payload_com[i] != 0.0) return false;
    for (int i = 0; i < 9; ++i) if (I[i] != 0.0) return false;
  }
  return true;
}

// The ranges of hunter_b200.h's hb_terrain: grid sizes, a finite origin, a finite positive spacing, finite heights where they are read
static bool terrain_ok(const hb_terrain& t) {
  if (t.nx < 2 || t.nx > HB_TERRAIN_MAX || t.ny < 2 || t.ny > HB_TERRAIN_MAX) return false;
  if (!isfinite(t.origin[0]) || !isfinite(t.origin[1]) || !isfinite(t.spacing) || !(t.spacing > 0.0)) return false;
  for (int j = 0; j < t.ny; ++j)
    for (int i = 0; i < t.nx; ++i) if (!isfinite(t.height[j][i])) return false;
  return true;
}

static bool push_schedule_ok(const hb_push_schedule& s) {
  if (s.n_push < 0 || s.n_push > HB_MAX_PUSHES) return false;
  for (int j = 0; j < s.n_push; ++j) {
    if (!isfinite(s.t_start[j]) || !isfinite(s.duration[j]) || !(s.duration[j] >= 0.0)) return false;
    for (int c = 0; c < 3; ++c) if (!isfinite(s.force[j][c]) || !isfinite(s.torque[j][c])) return false;
  }
  return true;
}

int hb_rollout_set_pushes(hb_ctx* ctx, int B, const hb_push_schedule* p) { return set_instances(ctx, B, p, push_schedule_ok, &hb_ctx::pushes); }
int hb_rollout_set_plant_variations(hb_ctx* ctx, int B, const hb_plant_variation* v) {
  return set_instances(ctx, B, v, plant_variation_ok, &hb_ctx::variations);
}
int hb_rollout_set_terrains(hb_ctx* ctx, int B, const hb_terrain* t) { return set_instances(ctx, B, t, terrain_ok, &hb_ctx::terrains); }

// The ranges of hunter_b200.h's hb_goal_schedule: the count, finite times in ascending order, finite goals
static bool goal_schedule_ok(const hb_goal_schedule& s) {
  if (s.n_goal < 0 || s.n_goal > HB_MAX_GOALS) return false;
  for (int j = 0; j < s.n_goal; ++j) {
    if (!isfinite(s.time[j]) || (j > 0 && s.time[j] < s.time[j - 1])) return false;
    for (int c = 0; c < 3; ++c) if (!isfinite(s.goal[j][c])) return false;
  }
  return true;
}

// The captured goals, allocated at max_batch by their first use (hb_rollout_set_goals with schedules, hb_episode_restore)
static int goal_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->goal_mem, [&](void* m) {
    size_t off = 0;
    ctx->goal_tg = carve<hb_target>(m, off, Bc); ctx->goal_idx = carve<int32_t>(m, off, Bc);
    return off;
  });
}

int hb_rollout_set_goals(hb_ctx* ctx, int B, const hb_goal_schedule* g) {
  int rc = set_instances(ctx, B, g, goal_schedule_ok, &hb_ctx::goals);
  if (rc || ctx->goals.n == 0) return rc;
  rc = goal_reserve(ctx);
  if (rc) { ctx->goals.n = 0; return rc; }
  CK(cudaMemsetAsync(ctx->goal_idx, 0xff, sizeof(int32_t) * ctx->cfg.max_batch, ctx->stream));     // every captured goal forgotten: index -1
  return HB_OK;
}

// The ranges of hunter_b200.h's hb_target: the sample count, strictly ascending finite times, finite states in the used samples
static bool target_ok(const hb_target& tg) {
  if (tg.n < 1 || tg.n > HB_MAX_TARGETS) return false;
  for (int k = 0; k < tg.n; ++k) {
    if (!isfinite(tg.time[k]) || (k > 0 && !(tg.time[k] > tg.time[k - 1]))) return false;
    for (int i = 0; i < 22; ++i) if (!isfinite(tg.state[k][i])) return false;
  }
  return true;
}

int hb_plan_set_targets(hb_ctx* ctx, int B, const hb_target* t) { return set_instances(ctx, B, t, target_ok, &hb_ctx::plan_targets); }

int hb_plan_set_settings(hb_ctx* ctx, int B, const hb_planner_settings* s) {
  return set_instances(ctx, B, s, planner_settings_ok, &hb_ctx::plan_settings);
}

static bool latency_ok(const int32_t& d) { return d >= 0; }     // the upper bound is the episode's mpc_every, checked by the episode call

int hb_rollout_set_mpc_latencies(hb_ctx* ctx, int B, const int32_t* ticks) { return set_instances(ctx, B, ticks, latency_ok, &hb_ctx::latencies); }

// The ranges of hunter_b200.h's hb_odometry_setting
static bool odometry_ok(const hb_odometry_setting& s) {
  if (s.period_ticks < 0 || s.delay_ticks < 0 || s.delay_ticks > HB_ODOM_MAX_DELAY) return false;
  for (double sigma : {s.sigma_position, s.sigma_drift}) if (!(sigma >= 0.0) || !isfinite(sigma)) return false;
  return true;
}

// The cameras' state, allocated at max_batch by its first use (hb_rollout_set_odometry with cameras, hb_episode_restore)
static int camera_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->odom_mem, [&](void* m) {
    size_t off = 0;
    ctx->odom_cam = carve<OdomCamera>(m, off, Bc);
    return off;
  });
}

int hb_rollout_set_odometry(hb_ctx* ctx, int B, const hb_odometry_setting* s) {
  int rc = set_instances(ctx, B, s, odometry_ok, &hb_ctx::odometry);
  if (rc || ctx->odometry.n == 0) return rc;
  rc = camera_reserve(ctx);
  if (rc) { ctx->odometry.n = 0; return rc; }
  CK(cudaMemsetAsync(ctx->odom_cam, 0, sizeof(OdomCamera) * ctx->cfg.max_batch, ctx->stream));     // every camera's history and bias cleared
  return HB_OK;
}

// The ranges of hunter_b200.h's hb_controller_setting: hb_wbc_set_settings' rules, every field finite, task gains and PD gains >= 0
static bool controller_setting_ok(const hb_controller_setting& s) {
  const double* f = reinterpret_cast<const double*>(&s);
  static_assert(sizeof(hb_controller_setting) == 26 * sizeof(double), "hb_controller_setting holds 26 doubles");
  for (int i = 0; i < 26; ++i) if (!isfinite(f[i])) return false;
  const hb_wbc_settings& w = s.wbc;
  for (double lim : w.torque_limits) if (!(lim > 0.0)) return false;
  if (!(w.friction_coefficient > 0.0) || !(w.weight_swing_leg > 0.0) || !(w.weight_base_accel > 0.0) || !(w.weight_contact_force >= 0.0)) return false;
  for (double k : {w.swing_kp, w.swing_kd, w.base_accel_kp, w.base_accel_kd, w.base_height_kp, w.base_height_kd, w.base_angular_kp, w.base_angular_kd})
    if (!(k >= 0.0)) return false;
  const hb_pd_gains& g = s.gains;
  for (double k : {g.kp_position, g.kd_position, g.kp_big_stance, g.kp_big_swing, g.kd_big, g.kp_small_stance, g.kp_small_swing, g.kd_small, g.kd_feet})
    if (!(k >= 0.0)) return false;
  return true;
}

int hb_rollout_set_controller_settings(hb_ctx* ctx, int B, const hb_controller_setting* s) {
  return set_instances(ctx, B, s, controller_setting_ok, &hb_ctx::controllers);
}

int hb_check_setting_records(int32_t kind, int B, const void* records, int32_t* first_bad) {
  if (!first_bad) return HB_EINVAL;
  *first_bad = -1;
  if (B < 0 || (B > 0 && !records)) return HB_EINVAL;
  switch (kind) {
    case HB_SETTING_PUSHES: return check_records(B, records, push_schedule_ok, first_bad);
    case HB_SETTING_PLANT_VARIATIONS: return check_records(B, records, plant_variation_ok, first_bad);
    case HB_SETTING_TERRAINS: return check_records(B, records, terrain_ok, first_bad);
    case HB_SETTING_GOALS: return check_records(B, records, goal_schedule_ok, first_bad);
    case HB_SETTING_ODOMETRY: return check_records(B, records, odometry_ok, first_bad);
    case HB_SETTING_CONTROLLERS: return check_records(B, records, controller_setting_ok, first_bad);
    case HB_SETTING_HARDWARE: return check_records(B, records, hardware_setting_ok, first_bad);
    case HB_SETTING_PLANNER: return check_records(B, records, planner_settings_ok, first_bad);
    case HB_SETTING_TARGETS: return check_records(B, records, target_ok, first_bad);
    case HB_SETTING_LATENCIES: return check_records(B, records, latency_ok, first_bad);
    default: return HB_EINVAL;
  }
}

// The camera read of a call whose instances start at ctx->base, on the context's odometry setting, its messages written to pos / has
static OdomRead odometry_read(const hb_ctx* ctx, double* pos, uint8_t* has) {
  const InstanceView<hb_odometry_setting> set = ctx->odometry.view(ctx->base);
  return OdomRead{set, set.recs ? ctx->odom_cam + ctx->base : nullptr, pos, has};
}

// The adopted policy ctx->pol, allocated at max_batch by its first use (hb_policy_update, an episode with a latency set)
static int policy_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  const int rc = reserve_group(&ctx->pol_mem, [&](void* m) {
    size_t off = 0;
    ctx->pol = carve_solution(m, off, Bc, ctx->cfg.horizon_N);
    return off;
  });
  if (rc) return rc;
  if (ctx->pol_have.size() != Bc) {
    try { ctx->pol_have.assign(Bc, 0); } catch (const std::bad_alloc&) { return HB_ENOMEM; }
  }
  return HB_OK;
}

// true when instances [lo, hi) have all adopted a policy
static bool policies_adopted(const hb_ctx* ctx, size_t lo, size_t hi) {
  if (hi > ctx->pol_have.size()) return false;
  for (size_t i = lo; i < hi; ++i) if (!ctx->pol_have[i]) return false;
  return true;
}

// policy_adopt_kernel on instances [0, B) after the entry checks: with lat set the episodes' rule at `tick`, otherwise the update mask
static int policy_adopt(hb_ctx* ctx, int B, InstanceView<int32_t> lat, long long tick, int every, const uint8_t* update) {
  const int rc = policy_reserve(ctx);
  if (rc) return rc;
  const size_t N = ctx->cfg.horizon_N, o = (size_t)ctx->base;
  const bool grid = ctx->cfg.event_nodes != 0;
  const int wpb = 4;
  return launch(ctx, K_UNPROFILED, policy_adopt_kernel, (B + wpb - 1) / wpb, 32 * wpb, 0, B, (int)N, lat, tick, every, update, rows_at(ctx->res, o, N, grid),
                rows_at(ctx->pol, o, N, grid));
}

// hb_resident_wbc_batch_dev; no_prev = true: the fallback has no previous solution yet (first tick after a cold start whose cycle ran no WBC).
// adopted: the adopted policy is evaluated instead of the resident solution (hb_policy_wbc_async); choice (the episodes): per instance one of
// the two (PolicyChoice); cs (the episodes): each instance's controller setting.
static int resident_wbc_impl(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                             int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status, bool no_prev, bool adopted = false,
                             const PolicyChoice& choice = PolicyChoice{}, ControllerView cs = ControllerView{}) {
  ENTER(ctx, B, t_now && rbd && x_des && u_des && mode_out && wbc_sol, UNCAPPED, [&] {   // a solution to evaluate
    return adopted ? policies_adopted(ctx, (size_t)ctx->base, (size_t)ctx->base + B) : ctx->base + B <= ctx->res_valid;
  });
  const size_t N = ctx->cfg.horizon_N;   // adopted: policies_adopted() passed, so the adopted rows are allocated
  const SolutionRows s = rows_at(adopted ? ctx->pol : ctx->res, (size_t)ctx->base, N, ctx->cfg.event_nodes != 0);
  const int wpb = 4;
  int rc = launch(ctx, K_UNPROFILED, policy_eval_kernel, (B + wpb - 1) / wpb, 32 * wpb, 0, B, (int)N, ctx->cfg.dt, 0.0, s, x_des, u_des, mode_out, t_now,
                  choice);
  if (!rc) rc = controller_wbc_dev(ctx, B, x_des, u_des, rbd, mode_out, stance_mode, wbc_sol, wbc_status, cs);
  if (!rc && torque) rc = launch(ctx, K_UNPROFILED, torque_kernel, (B * NJ + 127) / 128, 128, 0, B, wbc_sol, torque);
  return rc ? rc : wbc_fallback(ctx, B, no_prev, wbc_status, wbc_sol, torque);
}

int hb_resident_wbc_batch_dev(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                              int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status) {
  return resident_wbc_impl(ctx, B, t_now, rbd, stance_mode, x_des, u_des, mode_out, wbc_sol, torque, wbc_status, false);
}

int hb_policy_wbc_async(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                        int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status) {
  return resident_wbc_impl(ctx, B, t_now, rbd, stance_mode, x_des, u_des, mode_out, wbc_sol, torque, wbc_status, false, true);
}

// hb_joint_command_batch_dev, with each instance of `cs` on its own gains (the episodes)
static int joint_command_dev(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                             const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop, double* command,
                             double* output_torque, ControllerView cs) {
  ENTER(ctx, B, gains && x_des && u_des && wbc_sol && mode_cmd && rbd && command && output_torque, UNCAPPED);
  return launch(ctx, K_UNPROFILED, joint_command_kernel, (B + 63) / 64, 64, 0, B, *gains, cs, period, x_des, u_des, wbc_sol, mode_cmd, rbd, loaded,
                estop, command, output_torque);
}

int hb_default_rollout_params(hb_rollout_params* p) {
  if (!p) return HB_EINVAL;
  memset(p, 0, sizeof(*p));
  p->period = 0.002; p->mpc_every = 5; p->actuation_delay = 0.009;
  hb_default_sim_params(&p->sim);
  hb_default_pd_gains(&p->gains);
  for (int j = 0; j < NJ; ++j) p->torque_limit[j] = HB_WBC_TORQUE_LIMITS[j % 5];
  return HB_OK;
}

// hb_rollout_batch_dev's scratch, at max_batch
static int rollout_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->ro_mem, [&](void* m) {
    size_t off = 0;
    ctx->ro_cmd = carve<hb_rollout_command>(m, off, Bc); ctx->ro_in = carve<hb_plan_input>(m, off, Bc); ctx->ro_refs = carve<hb_reference>(m, off, Bc);
    ctx->ro_info = carve<hb_solve_info>(m, off, Bc); ctx->ro_pstat = carve<int32_t>(m, off, Bc); ctx->ro_t0 = carve<double>(m, off, Bc);
    ctx->ro_x0 = carve<double>(m, off, Bc * NX); ctx->ro_feet = carve<double>(m, off, Bc * 12); ctx->ro_sol = carve<double>(m, off, Bc * NWBC);
    ctx->ro_jcmd = carve<double>(m, off, Bc * NJ * 5); ctx->ro_jtau = carve<double>(m, off, Bc * NJ); ctx->ro_tau = carve<double>(m, off, Bc * NJ);
    ctx->ro_held = carve<double>(m, off, Bc * 32); ctx->ro_tnow = carve<double>(m, off, Bc); ctx->ro_wrench = carve<double>(m, off, Bc * 6);
    ctx->ro_cforce = carve<double>(m, off, Bc * 12); ctx->ro_cflag = carve<uint8_t>(m, off, Bc * 4);
    return off;
  });
}

// hb_rollout_estimated_batch_dev's scratch, at max_batch
static int estimation_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->re_mem, [&](void* m) {
    size_t off = 0;
    ctx->re_quat = carve<double>(m, off, Bc * 4); ctx->re_gyro = carve<double>(m, off, Bc * 3); ctx->re_acc = carve<double>(m, off, Bc * 3);
    ctx->re_jpos = carve<double>(m, off, Bc * NJ); ctx->re_jvel = carve<double>(m, off, Bc * NJ); ctx->re_rbd = carve<double>(m, off, Bc * 32);
    ctx->re_flag = carve<uint8_t>(m, off, Bc * 4);
    ctx->re_opos = carve<double>(m, off, Bc * 3); ctx->re_ohas = carve<uint8_t>(m, off, Bc);
    return off;
  });
}

// the estimation arguments of an estimated episode; a null pointer to them is hb_rollout_batch_dev
struct EstimationArgs {
  const hb_estimation_params* ep;
  hb_estimation_state* est;
  hb_estimation_stats* stats;   // nullable
  double* log;                  // nullable
};

// The episode loop of hb_rollout_batch_dev (e == nullptr: exactly its launches) and hb_rollout_estimated_batch_dev
static int rollout_impl(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_rollout_command* cmd, double* rbd,
                        hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats, double* log, const EstimationArgs* e) {
  const bool params_ok = p && p->mpc_every >= 1 && p->period > 0.0 && p->log_every >= 0 && delay_ok(p->actuation_delay) && sim_params_ok(p->sim) &&
                         tick0 + n_ticks <= INT32_MAX && (!e || (e->ep && e->est && sensor_noise_ok(e->ep->noise)));
  const bool cold = tick0 == 0;
  // the MPC latencies of this batch's instances (hb_rollout_set_mpc_latencies): instances i < with_lat have one
  const InstanceSetting<int32_t>& lat = ctx->latencies;
  const int with_lat = std::min(lat.n, B);
  const int n_rows = (p && p->log_every > 0) ? (n_ticks + p->log_every - 1) / p->log_every : 0;   // rows of log and of the channels
  ENTER(ctx, B, n_ticks >= 0 && tick0 >= 0 && cmd && rbd && act && estop && stats && params_ok, CAPPED, [&] {
    for (const auto& ch : ctx->channels) if (p->log_every > 0 && ch.B > 0 && (ch.B < B || ch.rows < n_rows)) return false;
    for (int i = 0; i < B; ++i) {
      const hb_rollout_command& c = cmd[i];
      if (c.gait < 0 || c.gait > 3 || c.n_cmd < 1 || c.n_cmd > HB_ROLLOUT_MAX_CMDS || !(c.gait_start == c.gait_start)) return false;
      for (int k = 0; k < c.n_cmd; ++k) if (!(c.cmd_time[k] == c.cmd_time[k]) || (k > 0 && c.cmd_time[k] < c.cmd_time[k - 1])) return false;
    }
    for (int i = 0; i < lat.n; ++i) if (lat.host[i] > p->mpc_every) return false;     // latencies beyond one MPC period
    // a warm start continues from the resident solution, and the instances with a latency from their adopted policies
    for (int i = 0; i < with_lat && !cold; ++i) if (lat.host[i] >= 1 && !policies_adopted(ctx, i, i + 1)) return false;
    return cold || ctx->res_valid >= B;
  });
  if (n_ticks == 0) return HB_OK;
  int rc = rollout_reserve(ctx);
  if (!rc && e) rc = estimation_reserve(ctx);
  if (rc) return rc;
  // With a latency >= 1 in the batch: first_due[r] is the smallest latency d >= 1 with d % mpc_every == r (INT_MAX: none), so that some
  // instance adopts on tick a iff a >= first_due[a % mpc_every]; the policy evaluation chooses per instance (PolicyChoice).
  std::vector<int> first_due;
  PolicyChoice choice{};
  for (int i = 0; i < with_lat; ++i) {
    const int d = lat.host[i];
    if (d < 1) continue;
    if (first_due.empty()) first_due.assign(p->mpc_every, INT_MAX);
    first_due[d % p->mpc_every] = std::min(first_due[d % p->mpc_every], d);
  }
  const bool delayed = !first_due.empty();
  if (delayed) {
    rc = policy_reserve(ctx);
    if (rc) return rc;
    choice = PolicyChoice{lat.view(), rows_at(ctx->pol, 0, ctx->cfg.horizon_N, ctx->cfg.event_nodes != 0)};
  }
  CK(cudaMemcpyAsync(ctx->ro_cmd, cmd, sizeof(hb_rollout_command) * B, cudaMemcpyHostToDevice, ctx->stream));
  const double horizon = (ctx->cfg.event_nodes && ctx->cfg.time_horizon > 0.0) ? ctx->cfg.time_horizon : ctx->cfg.horizon_N * ctx->cfg.dt;
  const int n_log = log ? n_rows : 0, n_est_log = (e && e->log) ? n_rows : 0;
  // the channels this call records (hb_rollout_set_channel): every set one on the logged ticks, the sensors only in estimated episodes
  RecordSlots rec{};
  for (int c = 0; c < HB_CHANNELS && n_rows; ++c) {
    if (ctx->channels[c].B == 0 || (c == HB_CHANNEL_SENSORS && !e)) continue;
    rec.channel[rec.n] = c; rec.first[rec.n] = rec.width;
    rec.stride[rec.n] = (size_t)ctx->channels[c].rows * CHANNEL_WIDTH[c];
    rec.n++; rec.width += CHANNEL_WIDTH[c];
  }
  const bool contacts = ctx->channels[HB_CHANNEL_CONTACT_FORCE].B > 0 || ctx->channels[HB_CHANNEL_CONTACT_FLAG].B > 0;
  RecordSources src{ctx->ro_tau, ctx->ro_jcmd, ctx->xdes, ctx->udes, ctx->ro_sol, ctx->ro_cforce, ctx->wmode, ctx->wstatus, ctx->ro_pstat,
                    ctx->ro_cflag, ctx->ro_info};
  if (e) { src.quat = ctx->re_quat; src.gyro = ctx->re_gyro; src.acc = ctx->re_acc; src.jpos = ctx->re_jpos; src.jvel = ctx->re_jvel; }
  const unsigned grid = (B + 63) / 64;
  // what the controllers measure: the true state, or the filter's estimate
  double* meas = e ? ctx->re_rbd : rbd;
  // the push wrench the begin kernel writes and the plant applies, none without schedules
  double* wrench = ctx->pushes.n > 0 ? ctx->ro_wrench : nullptr;
  const InstanceView<hb_target> goal_targets{ctx->goal_tg, ctx->goals.n};    // what the planner reads: the targets of the captured goals
  // the cameras the sensor read reads and the messages the filter fuses, none without an odometry setting
  const bool odom = e && ctx->odometry.n > 0;
  const OdomRead odom_read = odom ? odometry_read(ctx, ctx->re_opos, ctx->re_ohas) : OdomRead{};
  const ControllerView controllers = ctx->controllers.view();   // each instance's WBC settings and PD gains, none without a setting
  const HardwareView hardware = ctx->hardware.view();           // each instance's actuators and sensors, none without a setting
  for (int k = 0; k < n_ticks && !rc; ++k) {
    const int64_t a = tick0 + k;
    const double t = (double)a * p->period;           // a product, never an accumulated sum: a stepwise caller reproduces it exactly
    const bool mpc = a % p->mpc_every == 0, first_cold = cold && k == 0;
    double* log_row = (n_log && k % p->log_every == 0) ? log + (size_t)(k / p->log_every) * 32 : nullptr;
    const bool record = rec.n && k % p->log_every == 0;
    rc = launch(ctx, K_UNPROFILED, rollout_tick_begin_kernel, grid, 64, 0, B, (int)a, t, p->min_base_height, rbd, ctx->ro_held, stats, ctx->ro_tnow,
                log_row, (size_t)n_log * 32, ctx->pushes.view(), wrench, ctx->terrains.view());
    if (!rc && e) {
      // LeggedController::updateStateEstimation: sensors and contact flags at the previous observation's time, filter, observation step
      double* est_row = (n_est_log && k % p->log_every == 0) ? e->log + (size_t)(k / p->log_every) * 32 : nullptr;
      rc = launch(ctx, K_UNPROFILED, sensor_read_kernel, grid, 64, 0, B, e->ep->noise, hardware, (uint32_t)a, p->sim.dt, (double)(a - 1) * p->period, rbd,
                  e->est, ctx->re_quat, ctx->re_gyro, ctx->re_acc, ctx->re_jpos, ctx->re_jvel, ctx->re_flag, odom_read);
      if (!rc) rc = launch(ctx, K_UNPROFILED, odom ? kf_update_kernel<hb_estimation_state, true> : kf_update_kernel<hb_estimation_state, false>, B, 32,
                           sizeof(KfShared), B, e->ep->kf, p->period, e->est, ctx->re_quat, ctx->re_gyro, ctx->re_acc, ctx->re_jpos, ctx->re_jvel, ctx->re_flag,
                           meas, (const double*)ctx->re_opos, (const uint8_t*)ctx->re_ohas);
      if (!rc) rc = launch(ctx, K_UNPROFILED, est_observe_kernel, grid, 64, 0, B, rbd, meas, stats, e->est, e->stats, est_row, (size_t)n_est_log * 32);
    }
    // MPC_MRT_Interface::updatePolicy of the instances whose solution comes into force on this tick, before this tick's cycle
    if (!rc && delayed && a >= first_due[a % p->mpc_every]) rc = policy_adopt(ctx, B, lat.view(), a, p->mpc_every, nullptr);
    if (!rc && mpc) {
      if (first_cold) CK(cudaMemsetAsync(ctx->res_stance, 0, sizeof(double) * B * 12, ctx->stream));   // latestStanceposition_ starts at zero
      rc = launch(ctx, K_UNPROFILED, rollout_plan_inputs_kernel, grid, 64, 0, B, t, horizon, ctx->ro_cmd, meas, e ? e->est : nullptr, ctx->ro_in,
                  ctx->goals.view(), first_cold ? 1 : 0, ctx->goal_tg, ctx->goal_idx, plan_consts());
      if (!rc) rc = launch(ctx, K_UNPROFILED, plan_prepare_kernel, grid, 64, 0, B, ctx->ro_in, ctx->ro_t0, ctx->ro_x0, ctx->ro_feet);
      if (!rc) rc = plan_dev(ctx, B, ctx->ro_in, ctx->ro_feet, ctx->res_stance, ctx->ro_refs, ctx->ro_pstat, goal_targets, ctx->goal_idx,
                             ctx->plan_settings.view());
      if (!rc) rc = resident_cycle_impl(ctx, B, first_cold, 0.0, ctx->ro_t0, ctx->ro_x0, ctx->ro_refs, meas, ctx->ro_info, nullptr, nullptr, nullptr, false);
      // the cold tick: every instance with a latency starts with the policy of this first solve
      if (!rc && delayed && first_cold) {
        rc = policy_adopt(ctx, B, lat.view(), -1, p->mpc_every, nullptr);
        for (int i = 0; i < with_lat && !rc; ++i) if (lat.host[i] >= 1) ctx->pol_have[i] = 1;
      }
      if (!rc && e) rc = launch(ctx, K_UNPROFILED, est_schedule_kernel, grid, 64, 0, B, ctx->ro_refs, e->est);
    }
    // the cycle ran no WBC, so after a cold start the first tick's fallback has no previous solution, as the cycle's own would not have
    if (!rc) rc = resident_wbc_impl(ctx, B, ctx->ro_tnow, meas, nullptr, ctx->xdes, ctx->udes, ctx->wmode, ctx->ro_sol, nullptr, ctx->wstatus, first_cold,
                                    false, choice, controllers);
    if (!rc) rc = joint_command_dev(ctx, B, &p->gains, p->period, ctx->xdes, ctx->udes, ctx->ro_sol, ctx->wmode, meas, nullptr, estop, ctx->ro_jcmd,
                                    ctx->ro_jtau, controllers);
    if (!rc) rc = actuation_dev(ctx, B, p->actuation_delay, hardware, ctx->ro_tnow, act, ctx->ro_jcmd, rbd, ctx->ro_tau);
    if (!rc) rc = launch(ctx, K_UNPROFILED, rollout_saturate_kernel, (B * NJ + 127) / 128, 128, 0, B, *p, hardware, ctx->ro_tau);
    if (!rc) rc = sim_step(ctx, B, p->sim, rbd, ctx->ro_tau, wrench, ctx->variations.view(), ctx->terrains.view(),
                           record && contacts ? ctx->ro_cforce : nullptr, record && contacts ? ctx->ro_cflag : nullptr);
    if (!rc && record) {
      for (int j = 0; j < rec.n; ++j)
        rec.dst[j] = static_cast<char*>(ctx->channels[rec.channel[j]].buf) + (size_t)(k / p->log_every) * CHANNEL_WIDTH[rec.channel[j]] * CHANNEL_BYTES[rec.channel[j]];
      src.mpc = mpc ? 1 : 0;
      rc = launch(ctx, K_UNPROFILED, rollout_record_kernel, (unsigned)(((size_t)B * rec.width + 127) / 128), 128, 0, B, rec, src);
    }
    if (!rc) rc = launch(ctx, K_UNPROFILED, rollout_tick_end_kernel, grid, 64, 0, B, (int)a, mpc ? 1 : 0, ctx->ro_info, ctx->ro_pstat, ctx->wstatus, estop, ctx->ro_tau, ctx->ro_held, rbd, stats);
  }
  return rc;
}

int hb_rollout_batch_dev(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_rollout_command* cmd, double* rbd,
                         hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats, double* log) {
  return rollout_impl(ctx, B, tick0, n_ticks, p, cmd, rbd, act, estop, stats, log, nullptr);
}

int hb_rollout_estimated_batch_dev(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_estimation_params* ep,
                                   const hb_rollout_command* cmd, double* rbd, hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats,
                                   hb_estimation_state* est, hb_estimation_stats* est_stats, double* log, double* est_log) {
  const EstimationArgs e{ep, est, est_stats, est_log};
  return rollout_impl(ctx, B, tick0, n_ticks, p, cmd, rbd, act, estop, stats, log, &e);
}

int hb_rollout_set_channel(hb_ctx* ctx, int32_t channel, int B, int rows, void* buffer) {
  const int rc = enter(ctx, B, channel >= 0 && channel < HB_CHANNELS && rows >= 0 && (B == 0 || buffer), CAPPED);
  if (rc == EMPTY) { ctx->channels[channel] = {nullptr, 0, 0}; return HB_OK; }
  if (rc) return rc;
  ctx->channels[channel] = {buffer, B, rows};
  return HB_OK;
}

// ---------------------------------------------------------------------------------------------- episode snapshots
// The segments of a snapshot row (hunter_b200.h, "episode snapshots") over this context's buffers, in the row's order; head: the headers
// a save writes (null: a restore, which keeps the headers out of the context)
struct EpisodeTable {
  EpisodeSegments t{};
  uint32_t words = 0;
  void add(void* buf, size_t bytes, uint32_t fill = 0, bool by_row = false) {
    t.seg[t.n++] = EpisodeSegment{static_cast<char*>(buf), (uint32_t)bytes, words, fill, by_row ? 1 : 0};
    words += (uint32_t)((bytes + 7) / 8);
  }
  // the rows of a solution that the layout of this grid holds, in SolutionRows' order
  void add_solution(const SolutionRows& r, size_t N, bool grid) {
    add(r.t0, sizeof(double)); add(r.xt, sizeof(double) * (N + 1) * NX); add(r.ut, sizeof(double) * N * NU);
    if (grid) add(r.tk, sizeof(double) * (N + 1));
    add(r.mode, sizeof(int32_t) * (N + 1));
    if (grid) add(r.nn, sizeof(int32_t));
  }
};
static_assert(sizeof(hb_target) % 4 == 0 && sizeof(OdomCamera) % 4 == 0, "snapshot segments are copied in 4-byte units");

static EpisodeSegments episode_segments(const hb_ctx* ctx, int64_t* head) {
  const size_t N = ctx->cfg.horizon_N;
  const bool grid = ctx->cfg.event_nodes != 0;
  EpisodeTable e;
  e.add(head, HB_EPISODE_HEADER_BYTES, 0, true);
  e.add_solution(rows_at(ctx->res, 0, N, grid), N, grid);
  e.add(ctx->res_sol, sizeof(double) * NWBC);
  e.add(ctx->res_stance, sizeof(double) * 12);
  e.add(ctx->goal_idx, sizeof(int32_t), 0xffffffffu);       // unallocated: no goal captured
  e.add(ctx->goal_tg, sizeof(hb_target));
  e.add_solution(ctx->pol_mem ? rows_at(ctx->pol, 0, N, grid) : SolutionRows{}, N, grid);
  e.add(ctx->odom_cam, sizeof(OdomCamera));
  e.t.row_words = e.words;
  return e.t;
}

// The staging of the snapshot calls, at max_batch
static int snapshot_reserve(hb_ctx* ctx) {
  const size_t Bc = ctx->cfg.max_batch;
  return reserve_group(&ctx->snap_mem, [&](void* m) {
    size_t off = 0;
    ctx->snap_src = carve<int32_t>(m, off, Bc); ctx->snap_head = carve<int64_t>(m, off, Bc * 4);
    return off;
  });
}

// episode_copy_kernel over B rows, after the entry checks. src (host) is staged in stream order, so a later call's staging cannot overtake
// this call's kernel.
static int episode_copy(hb_ctx* ctx, int B, const int32_t* src, bool restore, const void* rows, int64_t* head) {
  if (src) CK(cudaMemcpyAsync(ctx->snap_src, src, sizeof(int32_t) * B, cudaMemcpyHostToDevice, ctx->stream));
  const EpisodeSegments t = episode_segments(ctx, head);
  const size_t n = (size_t)B * t.row_words;
  return launch(ctx, K_UNPROFILED, episode_copy_kernel, (unsigned)((n + 127) / 128), 128, 0, B, t, src ? (const int32_t*)ctx->snap_src : nullptr,
                restore ? 1 : 0, static_cast<uint32_t*>(const_cast<void*>(rows)));
}

int64_t hb_episode_state_bytes(const hb_ctx* ctx) { return ctx ? (int64_t)episode_segments(ctx, nullptr).row_words * 8 : HB_EINVAL; }

int hb_episode_save_async(hb_ctx* ctx, int B, const int32_t* src, void* rows) {
  ENTER(ctx, B, B == 0 || rows, CAPPED, [&] { return !src || std::all_of(src, src + B, [&](int32_t s) { return s >= 0 && s < ctx->cfg.max_batch; }); });
  int rc = snapshot_reserve(ctx);
  if (rc) return rc;
  std::vector<int64_t> head;
  try { head.resize((size_t)B * 4); } catch (const std::bad_alloc&) { return HB_ENOMEM; }
  const int64_t bytes = hb_episode_state_bytes(ctx);
  for (int i = 0; i < B; ++i) {
    const int s = src ? src[i] : i;
    const bool pol = (size_t)s < ctx->pol_have.size() && ctx->pol_have[s];
    int64_t* h = &head[(size_t)i * 4];
    h[0] = ctx->cfg.horizon_N; h[1] = ctx->cfg.event_nodes; h[2] = bytes;
    h[3] = (s < ctx->res_valid ? HB_EPISODE_HAS_SOLUTION : 0) | (s < ctx->res_sol_valid ? HB_EPISODE_HAS_FALLBACK : 0) | (pol ? HB_EPISODE_HAS_POLICY : 0);
  }
  CK(cudaMemcpyAsync(ctx->snap_head, head.data(), sizeof(int64_t) * head.size(), cudaMemcpyHostToDevice, ctx->stream));
  return episode_copy(ctx, B, src, false, rows, ctx->snap_head);
}

int hb_episode_restore(hb_ctx* ctx, int B, const int32_t* src, int n_rows, const void* rows) {
  ENTER(ctx, B, B == 0 || (rows && n_rows >= 1), CAPPED, [&] {
    return src ? std::all_of(src, src + B, [&](int32_t s) { return s >= 0 && s < n_rows; }) : B <= n_rows;
  });
  // the headers of the rows up to the last one restored, read back before anything changes
  const int n_head = src ? *std::max_element(src, src + B) + 1 : B;
  const int64_t bytes = hb_episode_state_bytes(ctx);
  std::vector<int64_t> head;
  try { head.resize((size_t)n_head * 4); } catch (const std::bad_alloc&) { return HB_ENOMEM; }
  CK(cudaMemcpy2DAsync(head.data(), HB_EPISODE_HEADER_BYTES, rows, (size_t)bytes, HB_EPISODE_HEADER_BYTES, n_head, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  // every row of this layout with a solution; k: the first restored instance without a fallback solution, after which none may have one
  int k = B;
  bool any_policy = false;
  for (int i = 0; i < B; ++i) {
    const int64_t* h = &head[(size_t)(src ? src[i] : i) * 4];
    if (h[0] != ctx->cfg.horizon_N || h[1] != ctx->cfg.event_nodes || h[2] != bytes || !(h[3] & HB_EPISODE_HAS_SOLUTION)) return HB_EINVAL;
    const bool fallback = (h[3] & HB_EPISODE_HAS_FALLBACK) != 0;
    if (!fallback && k == B) k = i;
    if (fallback && k < B) return HB_EINVAL;
    any_policy |= (h[3] & HB_EPISODE_HAS_POLICY) != 0;
  }
  if (k < B && ctx->res_sol_valid > B) return HB_EINVAL;     // instances beyond B keep a previous solution that instance k lacks
  // the buffers the rows write: the goal and camera state, and the adopted policy when a row holds one or the context has one
  int rc = snapshot_reserve(ctx);
  if (!rc) rc = goal_reserve(ctx);
  if (!rc) rc = camera_reserve(ctx);
  if (!rc && (any_policy || ctx->pol_mem)) rc = policy_reserve(ctx);
  if (!rc) rc = episode_copy(ctx, B, src, true, rows, nullptr);
  if (rc) return rc;
  ctx->res_valid = std::max(ctx->res_valid, B);
  ctx->res_sol_valid = k < B ? k : std::max(ctx->res_sol_valid, B);
  for (int i = 0; i < B && !ctx->pol_have.empty(); ++i) ctx->pol_have[i] = (head[(size_t)(src ? src[i] : i) * 4 + 3] & HB_EPISODE_HAS_POLICY) ? 1 : 0;
  CK(cudaStreamSynchronize(ctx->stream));
  return HB_OK;
}

int hb_default_estimation_params(hb_estimation_params* p) {
  if (!p) return HB_EINVAL;
  memset(p, 0, sizeof(*p));
  return hb_default_kf_params(&p->kf);
}

int hb_estimation_reset(int B, uint64_t first_stream, hb_estimation_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    memset(&state[i], 0, sizeof(hb_estimation_state));
    hb_kf_reset(1, &state[i].kf);
    state[i].noise_stream = first_stream + (uint64_t)i;
  }
  return HB_OK;
}

// hb_sim_read_sensors_batch_dev, with each instance of `hw` on its own sensors (hb_sim_read_sensors_hw)
static int read_sensors_dev(hb_ctx* ctx, int B, const hb_sensor_noise* noise, HardwareView hw, int64_t tick, double accel_dt, const double* rbd,
                            hb_estimation_state* est, double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos, double* joint_vel) {
  ENTER(ctx, B, noise && rbd && est && quat && ang_vel_local && lin_acc_local && joint_pos && joint_vel && sensor_noise_ok(*noise) && accel_dt > 0.0 &&
        tick >= 0 && tick <= UINT32_MAX, CAPPED);
  return launch(ctx, K_UNPROFILED, sensor_read_kernel, (B + 63) / 64, 64, 0, B, *noise, hw, (uint32_t)tick, accel_dt, 0.0, rbd, est, quat, ang_vel_local,
                lin_acc_local, joint_pos, joint_vel, (uint8_t*)nullptr, OdomRead{});
}

int hb_sim_read_sensors_batch_dev(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, double accel_dt, const double* rbd,
                                  hb_estimation_state* est, double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos,
                                  double* joint_vel) {
  return read_sensors_dev(ctx, B, noise, HardwareView{}, tick, accel_dt, rbd, est, quat, ang_vel_local, lin_acc_local, joint_pos, joint_vel);
}

int hb_sim_read_odometry_async(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, const double* rbd, const hb_estimation_state* est,
                               double* pos, uint8_t* has_msg) {
  ENTER(ctx, B, noise && rbd && est && pos && has_msg && tick >= 0 && tick <= UINT32_MAX, CAPPED);
  return launch(ctx, K_UNPROFILED, odometry_read_kernel, (B + 63) / 64, 64, 0, B, noise->seed, (uint32_t)tick, rbd, est, odometry_read(ctx, pos, has_msg));
}

int hb_observer_reset(int B, hb_observer_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  memset(state, 0, sizeof(hb_observer_state) * (size_t)B);      // pSCgZinvlast_ starts at zero (StateEstimateBase.cpp:58-59)
  return HB_OK;
}

int hb_contact_force_estimate_batch_dev(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                        const double* tau_cmd, double* est_contact_force, double* disturbance_torque) {
  ENTER(ctx, B, state && rbd && tau_cmd && est_contact_force && cutoff_ok(cutoff_frequency, dt), UNCAPPED);
  return launch(ctx, K_UNPROFILED, contact_force_kernel, B, 32, 0, B, cutoff_frequency, dt, state, rbd, tau_cmd, est_contact_force, disturbance_torque);
}

int hb_default_pd_gains(hb_pd_gains* g) {
  if (!g) return HB_EINVAL;
  g->kp_position = 10.0; g->kd_position = 3.0;
  g->kp_big_stance = 40.0; g->kp_big_swing = 30.0; g->kd_big = 2.0;
  g->kp_small_stance = 30.0; g->kp_small_swing = 20.0; g->kd_small = 2.0;
  g->kd_feet = 0.01;
  return HB_OK;
}

int hb_joint_command_batch_dev(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                               const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                               double* command, double* output_torque) {
  return joint_command_dev(ctx, B, gains, period, x_des, u_des, wbc_sol, mode_cmd, rbd, loaded, estop, command, output_torque, ControllerView{});
}

int hb_rbd_to_centroidal_batch_dev(hb_ctx* ctx, int B, const double* rbd, double* x) {
  ENTER(ctx, B, rbd && x, UNCAPPED);
  return launch(ctx, K_UNPROFILED, rbd_to_centroidal_kernel, (B + 63) / 64, 64, 0, B, rbd, x);
}

int hb_reference_expand_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref, int32_t* mode) {
  ENTER(ctx, B, t0 && refs && x_ref && swing_ref && mode, UNCAPPED);
  return launch(ctx, K_UNPROFILED, reference_expand_kernel, B, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, t0, refs, x_ref, swing_ref, mode, nullptr);
}

int hb_reference_expand_grid_batch_dev(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref,
                                       int32_t* mode) {
  ENTER(ctx, B, node_times && refs && x_ref && swing_ref && mode, UNCAPPED);
  return launch(ctx, K_UNPROFILED, reference_expand_kernel, B, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, nullptr, refs, x_ref, swing_ref, mode, node_times);
}

int hb_contact_positions_batch_dev(hb_ctx* ctx, int B, const double* x, double* pos) {
  ENTER(ctx, B, x && pos, UNCAPPED);
  return launch(ctx, K_UNPROFILED, contact_positions_kernel, (B + 63) / 64, 64, 0, B, x, pos);
}

int hb_probe_flow_map_dev(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  ENTER(ctx, B, x && u && f && A && Bm, UNCAPPED);
  return launch(ctx, K_UNPROFILED, probe_flow_map_kernel, B, 32, sizeof(ProbeShared), B, x, u, f, A, Bm, ee);
}

// ------------------------------------------------------------------------------------------ host-pointer entry points
// Each call checks its arguments, declares its host inputs and outputs to a Staging (per-instance element counts) and runs the
// device-pointer entry point on the staged slices.
#define H2D(dst, src, n) CK(cudaMemcpyAsync(dst, src, (n), cudaMemcpyHostToDevice, ctx->stream))
#define D2H(dst, src, n) CK(cudaMemcpyAsync(dst, src, (n), cudaMemcpyDeviceToHost, ctx->stream))

int hb_wbc_qp_batch(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                    double* x, int32_t* status, int32_t* iters) {
  ENTER(ctx, B, H && g && A && lbA && ubA && x, UNCAPPED, [&] { return qp_shape_ok(n, m); });
  Staging s(ctx, B);
  auto dH = s.in(H, (size_t)n * n); auto dA = s.in(A, (size_t)m * n); auto dg = s.in(g, n); auto dlb = s.in(lbA, m); auto dub = s.in(ubA, m);
  auto dx = s.out(x, n); auto dst = s.out(status, 1); auto dit = s.out(iters, 1);
  return s.run(1, [&](Chunk) { return hb_wbc_qp_batch_dev(ctx, B, n, m, dH, dg, dA, dlb, dub, dx, dst, dit); });
}

int hb_wbc_assemble_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                          const uint8_t* stance_mode, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_rows) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && H && g && A && lbA && ubA && m_rows, CAPPED);
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto sm = s.in_or_null(stance_mode, 1);
  auto dH = s.out(H, QP_STRIDE_H); auto dA = s.out(A, QP_STRIDE_A); auto dg = s.out(g, NWBC); auto dlb = s.out(lbA, WBC_ROWS);
  auto dub = s.out(ubA, WBC_ROWS); auto dm = s.out(m_rows, 1);
  return s.run(1, [&](Chunk) { return hb_wbc_assemble_batch_dev(ctx, B, xd, ud, r, md, sm, dH, dg, dA, dlb, dub, dm); });
}

int hb_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                       const uint8_t* stance_mode, double* sol, int32_t* status) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && sol, CAPPED);
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto sm = s.in_or_null(stance_mode, 1);
  auto dsol = s.out(sol, NWBC); auto dst = s.out(status, 1);
  return s.run(1, [&](Chunk) { return hb_wbc_solve_batch_dev(ctx, B, xd, ud, r, md, sm, dsol, dst); });
}

int hb_hoqp_solve_batch(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack, int32_t* status) {
  ENTER(ctx, B, problems && x, CAPPED, [&] {
    for (int i = 0; i < B; ++i) {
      const hb_hoqp_problem& p = problems[i];
      if (p.n < 1 || p.n > HB_HOQP_N || p.levels < 1 || p.levels > HB_HOQP_MAX_LEVELS) return false;
      int stk = 0;
      for (int l = 0; l < p.levels; ++l) { if (p.ma[l] < 0 || p.ma[l] > HB_HOQP_MAX_EQ || p.md[l] < 0 || p.md[l] > HB_HOQP_MAX_IN) return false; stk += p.md[l]; }
      if (stk > HB_HOQP_MAX_STACKED) return false;
    }
    return true;
  });
  Staging s(ctx, B);
  auto pb = s.in(problems, 1); auto dx = s.out(x, HQ_N); auto dsl = s.out(slack, HQ_STK); auto dst = s.out(status, 1);
  return s.run(1, [&](Chunk) { return hb_hoqp_solve_batch_dev(ctx, B, pb, dx, dsl, dst); });
}

int hb_hierarchical_wbc_tasks_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                    hb_hoqp_problem* problems) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && problems, CAPPED);
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto pb = s.out(problems, 1);
  return s.run(1, [&](Chunk) { return hwbc_tasks_dev(ctx, B, xd, ud, r, md, pb); });
}

int hb_hierarchical_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                                    int32_t* status) {
  ENTER(ctx, B, x_des && u_des && rbd && mode && sol, CAPPED);
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1);
  auto dsol = s.out(sol, NWBC); auto dst = s.out(status, 1);
  return s.run(1, [&](Chunk) { return hb_hierarchical_wbc_solve_batch_dev(ctx, B, xd, ud, r, md, dsol, dst); });
}

int hb_mpc_cold_start_batch(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj) {
  ENTER(ctx, B, x0 && mode && x_traj && u_traj, CAPPED);
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto md = s.in(mode, N + 1); auto xt = s.out(x_traj, (N + 1) * NX); auto ut = s.out(u_traj, N * NU);
  return s.run(1, [&](Chunk) { return hb_mpc_cold_start_batch_dev(ctx, B, d0, md, xt, ut); });
}

int hb_mpc_solve_batch(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode, double* x_traj,
                       double* u_traj, hb_solve_info* info) {
  ENTER(ctx, B, x0 && x_ref && swing_ref && mode && x_traj && u_traj, CAPPED);
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto inf = s.out(info, 1);
  return s.run(1, [&](Chunk) { return hb_mpc_solve_batch_dev(ctx, B, d0, xr, sw, md, xt, ut, inf); });
}

int hb_mpc_solve_grid_batch(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                            const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info) {
  ENTER(ctx, B, x0 && node_times && n_intervals && x_ref && swing_ref && mode && x_traj && u_traj, CAPPED, [&] {
    const size_t N = ctx->cfg.horizon_N;
    for (int i = 0; i < B; ++i) {      // a grid the kernels can walk: 1 <= n <= N intervals of positive length
      if (n_intervals[i] < 1 || n_intervals[i] > (int)N) return false;
      for (int k = 0; k < n_intervals[i]; ++k) if (!(node_times[(size_t)i * (N + 1) + k + 1] > node_times[(size_t)i * (N + 1) + k])) return false;
    }
    return true;
  });
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto tk = s.in(node_times, N + 1); auto nn = s.in(n_intervals, 1);
  auto inf = s.out(info, 1);
  return s.run(1, [&](Chunk) { return hb_mpc_solve_grid_batch_dev(ctx, B, d0, tk, nn, xr, sw, md, xt, ut, inf); });
}

int hb_time_grid_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals, int32_t* status) {
  ENTER(ctx, B, t0 && refs && node_times && n_intervals, CAPPED, [&] { return references_valid(B, refs); });
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto rf = s.in(refs, 1); auto tk = s.out(node_times, N + 1); auto nn = s.out(n_intervals, 1); auto st = s.out(status, 1);
  return s.run(1, [&](Chunk) { return hb_time_grid_batch_dev(ctx, B, d0, rf, tk, nn, st); });
}

int hb_reference_expand_grid_batch(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref,
                                   int32_t* mode) {
  ENTER(ctx, B, node_times && refs && x_ref && swing_ref && mode, CAPPED, [&] { return references_valid(B, refs); });
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto tk = s.in(node_times, N + 1); auto rf = s.in(refs, 1);
  auto xr = s.out(x_ref, (N + 1) * NX); auto sw = s.out(swing_ref, (N + 1) * 24); auto md = s.out(mode, N + 1);
  return s.run(1, [&](Chunk) { return hb_reference_expand_grid_batch_dev(ctx, B, tk, rf, xr, sw, md); });
}

int hb_resident_write_batch(hb_ctx* ctx, int B, const double* t0, const double* x_traj, const double* u_traj, const int32_t* mode, const double* node_times,
                            const int32_t* n_intervals) {
  ENTER(ctx, B, t0 && x_traj && u_traj, CAPPED, [&] {
    if (!ctx->cfg.event_nodes) return true;
    if (!node_times || !n_intervals) return false;      // an event-node context shifts between grids: the snapshot needs its grid
    for (int i = 0; i < B; ++i) if (n_intervals[i] < 1 || n_intervals[i] > ctx->cfg.horizon_N) return false;
    return true;
  });
  const bool grid = ctx->cfg.event_nodes != 0;
  const size_t N = ctx->cfg.horizon_N;
  const int rc = drain(ctx, [&]() -> int {
    const SolutionRows& r = ctx->res;
    H2D(r.t0, t0, sizeof(double) * B); H2D(r.xt, x_traj, sizeof(double) * B * (N + 1) * NX); H2D(r.ut, u_traj, sizeof(double) * B * N * NU);
    if (mode) H2D(r.mode, mode, sizeof(int32_t) * B * (N + 1));
    if (grid) { H2D(r.tk, node_times, sizeof(double) * B * (N + 1)); H2D(r.nn, n_intervals, sizeof(int32_t) * B); }
    return HB_OK;
  }());
  if (rc) return rc;
  if (ctx->res_valid < B) ctx->res_valid = B;
  return HB_OK;
}

int hb_resident_read_grid_batch(hb_ctx* ctx, int B, double* node_times, int32_t* n_intervals) {
  ENTER(ctx, B, node_times && n_intervals, UNCAPPED, [&] { return B <= ctx->res_valid && ctx->cfg.event_nodes; });
  const size_t N = ctx->cfg.horizon_N;
  return drain(ctx, [&]() -> int {
    D2H(node_times, ctx->res.tk, sizeof(double) * B * (N + 1)); D2H(n_intervals, ctx->res.nn, sizeof(int32_t) * B);
    return HB_OK;
  }());
}

int hb_control_step_batch(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                          const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                          int32_t* wbc_status) {
  ENTER(ctx, B, x0 && x_ref && swing_ref && mode && rbd && x_traj && u_traj, CAPPED);
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto r = s.in(rbd, 32);
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);
  // Two half-batches on two streams: the copies of one half overlap the kernels of the other (pinned host memory assumed).
  return s.run(B >= 256 ? 2 : 1, [&](Chunk k) {
    return hb_control_step_batch_dev(ctx, k.n, t_rel, d0.at(k.lo), xr.at(k.lo), sw.at(k.lo), md.at(k.lo), r.at(k.lo), xt.at(k.lo), ut.at(k.lo),
                                     inf.at(k.lo), sol.at(k.lo), tau.at(k.lo), st.at(k.lo));
  });
}

int hb_resident_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                            const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status) {
  ENTER(ctx, B, t0 && x0 && refs && rbd, CAPPED, [&] { return cold_start || ctx->res_valid >= B; });
  // a pinned (page-locked, mapped) reference array is read by the device directly
  const hb_reference* refs_dev = nullptr;
  {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, refs) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) refs_dev = static_cast<const hb_reference*>(at.devicePointer);
    else cudaGetLastError();
  }
  // Chunks on two streams, as in hb_control_step_batch; only the small per-instance inputs and results cross PCIe.
  // Automatic choice: with a pageable reference array the host packs the used entries, and from 4096 instances on two chunks hide that pass
  // and the copies behind the other chunk's kernels; below, the half-batch kernels of the sequential stages run no faster than the full
  // batch. With a pinned array there is no host pass to hide and one chunk is used at every size.
  const int nchunk = cycle_chunks(ctx, B, !refs_dev);
  // pinned path: validation and byte count happen on the device while it copies (no per-instance host work at all); the verdict, two words
  // per chunk {invalid structs, words read}, comes back with the results. Pageable path: the used entries are packed into the context's
  // pinned host buffer, copied, and unpacked on the device.
  size_t pack_words = 0;
  if (!refs_dev) {
    if (!references_valid(B, refs)) return HB_EINVAL;
    for (int i = 0; i < B; ++i) pack_words += ref_pack_words(refs[i]);
    pack_words += (size_t)B + 2 * (size_t)nchunk + 8;
  }
  const size_t stat_words = refs_dev ? 2 * (size_t)nchunk : 0;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto dx0 = s.in(x0, NX); auto r = s.in(rbd, 32); auto rf = s.tmp<hb_reference>(1);
  auto d_pack = s.buf<double>(pack_words); auto d_stat = s.buf<unsigned long long>(stat_words);
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);
  int rc = grow(ctx, &ctx->pinned, &ctx->pinned_cap, refs_dev ? sizeof(unsigned long long) * stat_words : sizeof(double) * pack_words, true);
  if (rc) return rc;
  double* h_pack = static_cast<double*>(ctx->pinned);
  unsigned long long* h_stat = static_cast<unsigned long long*>(ctx->pinned);
  size_t pack_base = 0;
  ctx->last_h2d_bytes = 0;
  rc = s.run(nchunk, [&](Chunk k) -> int {
    if (refs_dev) {
      CK(cudaMemsetAsync(d_stat.at(2 * k.c), 0, 2 * sizeof(unsigned long long), ctx->stream));
      const int r2 = launch(ctx, K_UNPROFILED, reference_gather_pinned_kernel, k.n, 128, 0, k.n, refs_dev + k.lo, rf.at(k.lo), d_stat.at(2 * k.c));
      if (r2) return r2;
      D2H(h_stat + 2 * k.c, d_stat.at(2 * k.c), 2 * sizeof(unsigned long long));
    } else {
      const size_t words = ref_pack(refs, k.lo, k.hi, h_pack + pack_base);
      H2D(d_pack.at(pack_base), h_pack + pack_base, sizeof(double) * words);
      const int r2 = launch(ctx, K_UNPROFILED, reference_unpack_kernel, k.n, 128, 0, k.n, reinterpret_cast<const long long*>(d_pack.at(pack_base)),
                            d_pack.at(pack_base), rf.at(k.lo));
      if (r2) return r2;
      pack_base += words;
      ctx->last_h2d_bytes += sizeof(double) * words;
    }
    return hb_resident_cycle_batch_dev(ctx, k.n, cold_start, t_rel, d0.at(k.lo), dx0.at(k.lo), rf.at(k.lo), r.at(k.lo), inf.at(k.lo), sol.at(k.lo),
                                       tau.at(k.lo), st.at(k.lo));
  });
  if (rc) return rc;
  if (refs_dev) {
    unsigned long long invalid = 0, words = 0;
    for (int c = 0; c < nchunk; ++c) { invalid += h_stat[2 * c]; words += h_stat[2 * c + 1]; }
    ctx->last_h2d_bytes = sizeof(double) * (size_t)words;
    if (invalid) { ctx->res_valid = 0; return HB_EINVAL; }      // malformed structs: counts were clamped on the device, the outputs are not meaningful
  }
  return HB_OK;
}

int hb_plan_references_gpu(hb_ctx* ctx, int B, const hb_plan_input* in, double* latest_stance, hb_reference* out, int32_t* status) {
  ENTER(ctx, B, in && latest_stance && out, CAPPED);
  Staging s(ctx, B);
  auto din = s.in(in, 1); auto ls = s.inout(latest_stance, 12); auto dout = s.out(out, 1); auto st = s.out(status, 1);
  return s.run(1, [&](Chunk) { return hb_plan_references_batch_dev(ctx, B, din, nullptr, ls, dout, st); });
}

int hb_resident_plan_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const hb_plan_input* in, const double* rbd, hb_solve_info* info,
                                 double* wbc_sol, double* torque, int32_t* wbc_status, int32_t* plan_status) {
  ENTER(ctx, B, in && rbd, CAPPED, [&] { return cold_start || ctx->res_valid >= B; });
  const int nchunk = cycle_chunks(ctx, B, true);
  Staging s(ctx, B);
  auto din = s.in(in, 1); auto r = s.in(rbd, 32);
  auto d0 = s.tmp<double>(1); auto dx0 = s.tmp<double>(NX); auto feet = s.tmp<double>(12); auto rf = s.tmp<hb_reference>(1);   // planner -> cycle
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1); auto pst = s.out(plan_status, 1);
  return s.run(nchunk, [&](Chunk k) -> int {
    const size_t lo = k.lo;
    const int n = k.n;
    if (cold_start) CK(cudaMemsetAsync(ctx->res_stance + lo * 12, 0, sizeof(double) * n * 12, ctx->stream));   // latestStanceposition_ starts at zero
    int r2 = launch(ctx, K_UNPROFILED, plan_prepare_kernel, (n + 63) / 64, 64, 0, n, din.at(lo), d0.at(lo), dx0.at(lo), feet.at(lo));
    if (!r2) r2 = hb_plan_references_batch_dev(ctx, n, din.at(lo), feet.at(lo), ctx->res_stance + lo * 12, rf.at(lo), pst.at(lo));
    if (!r2) r2 = hb_resident_cycle_batch_dev(ctx, n, cold_start, t_rel, d0.at(lo), dx0.at(lo), rf.at(lo), r.at(lo), inf.at(lo), sol.at(lo), tau.at(lo), st.at(lo));
    return r2;
  });
}

int hb_resident_read_batch(hb_ctx* ctx, int B, double* t0, double* x_traj, double* u_traj) {
  ENTER(ctx, B, true, UNCAPPED, [&] { return B <= ctx->res_valid; });
  const size_t N = ctx->cfg.horizon_N;
  return drain(ctx, [&]() -> int {
    if (t0) D2H(t0, ctx->res.t0, sizeof(double) * B);
    if (x_traj) D2H(x_traj, ctx->res.xt, sizeof(double) * B * (N + 1) * NX);
    if (u_traj) D2H(u_traj, ctx->res.ut, sizeof(double) * B * N * NU);
    return HB_OK;
  }());
}

int hb_joint_command_batch(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                           const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                           double* command, double* output_torque) {
  ENTER(ctx, B, gains && x_des && u_des && wbc_sol && mode_cmd && rbd && command && output_torque, CAPPED);
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto sol = s.in(wbc_sol, NWBC); auto md = s.in(mode_cmd, 1);
  auto ld = s.in_or_null(loaded, 1); auto es = s.inout_or_null(estop, 1); auto cmd = s.out(command, NJ * 5); auto tau = s.out(output_torque, NJ);
  return s.run(1, [&](Chunk) { return hb_joint_command_batch_dev(ctx, B, gains, period, xd, ud, sol, md, r, ld, es, cmd, tau); });
}

int hb_estimator_update_batch(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                              const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos, const double* joint_vel,
                              const uint8_t* contact_flag, double* rbd_out) {
  ENTER(ctx, B, params && state && quat && ang_vel_local && lin_acc_local && joint_pos && joint_vel && contact_flag && rbd_out, CAPPED);
  Staging s(ctx, B);
  auto kf = s.inout(state, 1); auto q = s.in(quat, 4); auto w = s.in(ang_vel_local, 3); auto a = s.in(lin_acc_local, 3);
  auto jp = s.in(joint_pos, NJ); auto jv = s.in(joint_vel, NJ); auto fl = s.in(contact_flag, 4); auto ro = s.out(rbd_out, 32);
  return s.run(1, [&](Chunk) { return hb_estimator_update_batch_dev(ctx, B, params, dt, kf, q, w, a, jp, jv, fl, ro); });
}

int hb_sim_read_sensors(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, double accel_dt, const double* rbd, hb_estimation_state* est,
                        double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos, double* joint_vel) {
  return hb_sim_read_sensors_hw(ctx, B, noise, nullptr, tick, accel_dt, rbd, est, quat, ang_vel_local, lin_acc_local, joint_pos, joint_vel);
}

// the one host-pointer sensor read: hb_sim_read_sensors is it with null records
int hb_sim_read_sensors_hw(hb_ctx* ctx, int B, const hb_sensor_noise* noise, const hb_hardware_setting* hw, int64_t tick, double accel_dt,
                           const double* rbd, hb_estimation_state* est, double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos,
                           double* joint_vel) {
  ENTER(ctx, B, noise && rbd && est && quat && ang_vel_local && lin_acc_local && joint_pos && joint_vel && sensor_noise_ok(*noise) && accel_dt > 0.0 &&
        tick >= 0 && tick <= UINT32_MAX, CAPPED, [&] { return all_ok(B, hw, hardware_setting_ok); });
  Staging s(ctx, B);
  auto r = s.in(rbd, 32); auto es = s.inout(est, 1); auto h = s.in_or_null(hw, 1); auto q = s.out(quat, 4); auto w = s.out(ang_vel_local, 3);
  auto a = s.out(lin_acc_local, 3); auto jp = s.out(joint_pos, NJ); auto jv = s.out(joint_vel, NJ);
  return s.run(1, [&](Chunk) { return read_sensors_dev(ctx, B, noise, {h, B}, tick, accel_dt, r, es, q, w, a, jp, jv); });
}

int hb_sim_read_odometry(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, const double* rbd, const hb_estimation_state* est,
                         double* pos, uint8_t* has_msg) {
  ENTER(ctx, B, noise && rbd && est && pos && has_msg && tick >= 0 && tick <= UINT32_MAX, CAPPED);
  Staging s(ctx, B);
  auto r = s.in(rbd, 32); auto es = s.in(est, 1); auto p = s.out(pos, 3); auto h = s.out(has_msg, 1);
  return s.run(1, [&](Chunk) { return hb_sim_read_odometry_async(ctx, B, noise, tick, r, es, p, h); });
}

int hb_estimator_fuse_odometry(hb_ctx* ctx, int B, const hb_kf_params* params, hb_kf_state* state, const double* pos, const uint8_t* has_msg,
                               const uint8_t* contact_flag, double* rbd) {
  ENTER(ctx, B, params && state && pos && has_msg && contact_flag && rbd, CAPPED);
  Staging s(ctx, B);
  auto st = s.inout(state, 1); auto p = s.in(pos, 3); auto h = s.in(has_msg, 1); auto fl = s.in(contact_flag, 4); auto r = s.inout(rbd, 32);
  return s.run(1, [&](Chunk) { return hb_estimator_fuse_odometry_async(ctx, B, params, st, p, h, fl, r); });
}

int hb_actuation_batch(hb_ctx* ctx, int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd,
                       double* tau) {
  return hb_actuation_hw(ctx, B, delay, nullptr, time, state, command, rbd, tau);
}

// the one host-pointer actuation: hb_actuation_batch is it with null records
int hb_actuation_hw(hb_ctx* ctx, int B, double delay, const hb_hardware_setting* hw, const double* time, hb_actuation_state* state, const double* command,
                    const double* rbd, double* tau) {
  ENTER(ctx, B, time && state && command && rbd && tau, CAPPED, [&] { return delay_ok(delay) && all_ok(B, hw, hardware_setting_ok); });
  Staging s(ctx, B);
  auto st = s.inout(state, 1); auto tm = s.in(time, 1); auto cmd = s.in(command, NJ * 5); auto r = s.in(rbd, 32); auto h = s.in_or_null(hw, 1);
  auto t = s.out(tau, NJ);
  return s.run(1, [&](Chunk) { return actuation_dev(ctx, B, delay, {h, B}, tm, st, cmd, r, t); });
}

int hb_sim_step_batch(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force, uint8_t* contact_flag) {
  return hb_sim_step_terrain(ctx, B, params, rbd, tau, nullptr, nullptr, nullptr, contact_force, contact_flag);
}

int hb_sim_step_wrench(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench, double* contact_force,
                       uint8_t* contact_flag) {
  return hb_sim_step_terrain(ctx, B, params, rbd, tau, wrench, nullptr, nullptr, contact_force, contact_flag);
}

int hb_sim_step_varied(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench, const hb_plant_variation* v,
                       double* contact_force, uint8_t* contact_flag) {
  return hb_sim_step_terrain(ctx, B, params, rbd, tau, wrench, v, nullptr, contact_force, contact_flag);
}

// the one host-pointer plant step: the three above are it with null terrains, variations and wrench
int hb_sim_step_terrain(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench, const hb_plant_variation* v,
                        const hb_terrain* ter, double* contact_force, uint8_t* contact_flag) {
  ENTER(ctx, B, params && rbd && tau, CAPPED,
        [&] { return sim_params_ok(*params) && all_ok(B, v, plant_variation_ok) && all_ok(B, ter, terrain_ok); });
  Staging s(ctx, B);
  auto r = s.inout(rbd, 32); auto t = s.in(tau, NJ); auto w = s.in_or_null(wrench, 6); auto pv = s.in_or_null(v, 1); auto pt = s.in_or_null(ter, 1);
  auto cf = s.out(contact_force, 12); auto fl = s.out(contact_flag, 4);
  return s.run(1, [&](Chunk) { return sim_step(ctx, B, *params, r, t, w, {pv, B}, {pt, B}, cf, fl); });
}

int hb_resident_wbc_batch(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                          int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status) {
  ENTER(ctx, B, t_now && rbd && x_des && u_des && mode_out && wbc_sol, CAPPED, [&] { return B <= ctx->res_valid; });
  Staging s(ctx, B);
  auto tn = s.in(t_now, 1); auto r = s.in(rbd, 32); auto sm = s.in_or_null(stance_mode, 1);
  auto xd = s.out(x_des, NX); auto ud = s.out(u_des, NU); auto md = s.out(mode_out, 1); auto sol = s.out(wbc_sol, NWBC);
  auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);    // always passed: the fallback and its bookkeeping run on every call
  return s.run(1, [&](Chunk) { return hb_resident_wbc_batch_dev(ctx, B, tn, r, sm, xd, ud, md, sol, tau, st); });
}

int hb_policy_update(hb_ctx* ctx, int B, const uint8_t* update) {
  ENTER(ctx, B, true, CAPPED, [&] {            // an instance that adopts needs a resident solution
    for (int i = 0; i < B; ++i) if ((!update || update[i]) && i >= ctx->res_valid) return false;
    return true;
  });
  Staging s(ctx, B);
  auto up = s.in_or_null(update, 1);
  const int rc = s.run(1, [&](Chunk) { return policy_adopt(ctx, B, {}, 0, 1, up); });
  if (rc) return rc;
  for (int i = 0; i < B; ++i) if (!update || update[i]) ctx->pol_have[i] = 1;
  return HB_OK;
}

int hb_policy_wbc(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des, int32_t* mode_out,
                  double* wbc_sol, double* torque, int32_t* wbc_status) {
  ENTER(ctx, B, t_now && rbd && x_des && u_des && mode_out && wbc_sol, CAPPED, [&] { return policies_adopted(ctx, 0, B); });
  Staging s(ctx, B);
  auto tn = s.in(t_now, 1); auto r = s.in(rbd, 32); auto sm = s.in_or_null(stance_mode, 1);
  auto xd = s.out(x_des, NX); auto ud = s.out(u_des, NU); auto md = s.out(mode_out, 1); auto sol = s.out(wbc_sol, NWBC);
  auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);    // always passed, as in hb_resident_wbc_batch
  return s.run(1, [&](Chunk) { return hb_policy_wbc_async(ctx, B, tn, r, sm, xd, ud, md, sol, tau, st); });
}

int hb_contact_force_estimate_batch(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                    const double* tau_cmd, double* est_contact_force, double* disturbance_torque) {
  ENTER(ctx, B, state && rbd && tau_cmd && est_contact_force, CAPPED, [&] { return cutoff_ok(cutoff_frequency, dt); });
  Staging s(ctx, B);
  auto st = s.inout(state, 1); auto r = s.in(rbd, 32); auto t = s.in(tau_cmd, NJ); auto est = s.out(est_contact_force, 16);
  auto dist = s.out(disturbance_torque, NQ);
  return s.run(1, [&](Chunk) { return hb_contact_force_estimate_batch_dev(ctx, B, cutoff_frequency, dt, st, r, t, est, dist); });
}

int hb_rbd_to_centroidal_batch(hb_ctx* ctx, int B, const double* rbd, double* x) {
  ENTER(ctx, B, rbd && x, CAPPED);
  Staging s(ctx, B);
  auto r = s.in(rbd, 32); auto dx = s.out(x, NX);
  return s.run(1, [&](Chunk) { return hb_rbd_to_centroidal_batch_dev(ctx, B, r, dx); });
}

int hb_reference_expand_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref, int32_t* mode) {
  ENTER(ctx, B, t0 && refs && x_ref && swing_ref && mode, CAPPED, [&] { return references_valid(B, refs); });
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto rf = s.in(refs, 1);
  auto xr = s.out(x_ref, (N + 1) * NX); auto sw = s.out(swing_ref, (N + 1) * 24); auto md = s.out(mode, N + 1);
  return s.run(1, [&](Chunk) { return hb_reference_expand_batch_dev(ctx, B, d0, rf, xr, sw, md); });
}

int hb_contact_positions_batch(hb_ctx* ctx, int B, const double* x, double* pos) {
  ENTER(ctx, B, x && pos, CAPPED);
  Staging s(ctx, B);
  auto dx = s.in(x, NX); auto dp = s.out(pos, 12);
  return s.run(1, [&](Chunk) { return hb_contact_positions_batch_dev(ctx, B, dx, dp); });
}

static std::atomic<int> g_plan_threads{0};   // 0 = hardware_concurrency (hb_plan_set_threads)
static int plan_range(int lo, int hi, const hb_plan_input* in, const hb_target* targets, const hb_planner_settings* settings, double* latest_stance,
                      hb_reference* out) {
  const hbplan::PlanConsts& pc = plan_consts();
  for (int i = lo; i < hi; ++i) {
    const int rc = hbplan::plan_one(pc, in[i], targets ? targets + i : nullptr, settings ? settings + i : nullptr, latest_stance + (size_t)i * 12,
                                    out + i, true);
    if (rc) return rc;
  }
  return HB_OK;
}

int hb_plan_set_threads(int n_threads) {
  if (n_threads < 0) return HB_EINVAL;
  g_plan_threads.store(n_threads);
  return HB_OK;
}

int hb_plan_references(int B, const hb_plan_input* in, double* latest_stance, hb_reference* out) {
  return hb_plan_references_targets(B, in, nullptr, latest_stance, out);
}

int hb_plan_references_targets(int B, const hb_plan_input* in, const hb_target* targets, double* latest_stance, hb_reference* out) {
  return hb_plan_references_settings(B, in, targets, nullptr, latest_stance, out);
}

int hb_plan_references_settings(int B, const hb_plan_input* in, const hb_target* targets, const hb_planner_settings* settings, double* latest_stance,
                                hb_reference* out) {
  if (B < 0 || !in || !latest_stance || !out || !all_ok(B, targets, target_ok) || !all_ok(B, settings, planner_settings_ok)) return HB_EINVAL;
  // instances are independent: spread them over the host cores (the planner feeds ~1e5 solves/s per GPU; one core plans ~2e4/s)
  unsigned hw = std::thread::hardware_concurrency();
  if (const int forced = g_plan_threads.load()) hw = (unsigned)forced;
  int nt = (int)std::min<unsigned>(hw ? hw : 1u, (unsigned)((B + 63) / 64));
  if (nt <= 1) return plan_range(0, B, in, targets, settings, latest_stance, out);
  std::vector<std::thread> pool;
  std::vector<int> rcs(nt, HB_OK);
  for (int t = 0; t < nt; ++t) {
    const int lo = (int)((long long)B * t / nt), hi = (int)((long long)B * (t + 1) / nt);
    pool.emplace_back([=, &rcs]() { rcs[t] = plan_range(lo, hi, in, targets, settings, latest_stance, out); });
  }
  for (auto& th : pool) th.join();
  for (int t = 0; t < nt; ++t) if (rcs[t]) return rcs[t];
  return HB_OK;
}

int hb_goal_to_target(int B, const double* t, const double* x, const double* goal, hb_target* out) {
  if (B < 0 || !t || !x || !goal || !out) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    const double* xi = x + (size_t)i * NX; const double* gi = goal + (size_t)i * 3;
    if (!isfinite(t[i]) || !isfinite(xi[6]) || !isfinite(xi[7]) || !isfinite(xi[8]) || !isfinite(xi[9]) || !isfinite(gi[0]) || !isfinite(gi[1]) ||
        !isfinite(gi[2]))
      return HB_EINVAL;
  }
  for (int i = 0; i < B; ++i) {
    memset(&out[i], 0, sizeof(hb_target));
    hbplan::goal_to_target(plan_consts(), t[i], x + (size_t)i * NX, goal + (size_t)i * 3, out[i]);
  }
  return HB_OK;
}

int hb_gait_select(int B, hb_gait_selector* state, const int32_t* gait_type, const double* cmd_vel, const double* target_state0, int32_t* level,
                   int32_t* insert) {
  if (B < 0 || !state || !gait_type || !cmd_vel || !target_state0 || !level || !insert) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    if (state[i].head < 0 || state[i].head >= 50 || state[i].count < 0 || state[i].count > 50) return HB_EINVAL;
    int ins = 0;
    level[i] = hbplan::gait_select(state + i, gait_type[i], cmd_vel + (size_t)i * 4, target_state0 + (size_t)i * 22, &ins);
    insert[i] = ins;
  }
  return HB_OK;
}

int hb_probe_flow_map(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  ENTER(ctx, B, x && u && f && A && Bm, CAPPED);
  Staging s(ctx, B);
  auto dx = s.in(x, NX); auto du = s.in(u, NU);
  auto df = s.out(f, NX); auto dA = s.out(A, TS); auto dB = s.out(Bm, TS); auto dee = s.out(ee, 24 + 36 * NX);
  return s.run(1, [&](Chunk) { return hb_probe_flow_map_dev(ctx, B, dx, du, df, dA, dB, dee); });
}

}  // extern "C"

#include "hb_shard.cuh"
