// The reference on the device: the packed upload of caller hb_reference structs (host packer and device unpacker), their validity
// rules (host check and the check fused into the pinned gather), the event-node time grid, the expansion onto the node grid, and
// the device planner (hb_planner.h compiled for the device).
#pragma once
#include "hb_common.cuh"
#include "hb_planner.h"     // also the C header (hb_reference) and <string.h> (the packer)
#include "hb_rbd.cuh"

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
// Packed upload of hb_reference (host-pointer cycle): only the used entries of the fixed-capacity struct cross PCIe (about 3 KB instead of
// 17.7 KB per instance). Stream layout per instance, 8-byte words: header {n_events, n_targets, n_segments[12], 2 pad} (8 words),
// event_times, modes (as int32 pairs, padded), target_times, target_states, segments. `offs` (B + 1 words offsets) leads the stream.
// ref_pack writes it on the host, reference_unpack_kernel reads it on the device.
struct RefPackHeader { int32_t n_events, n_targets, nseg[12], pad[2]; };
static_assert(sizeof(RefPackHeader) == 64, "header is 8 words");
__global__ void reference_unpack_kernel(int B, const long long* offs, const double* stream, hb_reference* refs) {
  const int inst = blockIdx.x;
  if (inst >= B) return;
  const double* p = stream + offs[inst];
  const RefPackHeader hd = *reinterpret_cast<const RefPackHeader*>(p);
  hb_reference& r = refs[inst];
  const int ne = min(max(hd.n_events, 0), HB_MAX_EVENTS), nt = min(max(hd.n_targets, 0), HB_MAX_TARGETS);
  p += 8;
  if (threadIdx.x == 0) { r.n_events = ne; r.n_targets = nt; for (int q = 0; q < 12; ++q) r.n_segments[q / 3][q % 3] = min(max(hd.nseg[q], 0), HB_MAX_SEGMENTS); }
  for (int i = threadIdx.x; i < ne; i += blockDim.x) r.event_times[i] = p[i];
  p += ne;
  const int32_t* pm = reinterpret_cast<const int32_t*>(p);
  for (int i = threadIdx.x; i <= ne; i += blockDim.x) r.modes[i] = pm[i];
  p += (ne + 2) / 2;
  for (int i = threadIdx.x; i < nt; i += blockDim.x) r.target_times[i] = p[i];
  p += nt;
  for (int i = threadIdx.x; i < nt * 22; i += blockDim.x) r.target_states[i / 22][i % 22] = p[i];
  p += nt * 22;
  for (int q = 0; q < 12; ++q) {
    const int ns = min(max(hd.nseg[q], 0), HB_MAX_SEGMENTS);
    double* dst = &r.segments[q / 3][q % 3][0][0];
    for (int i = threadIdx.x; i < ns * 6; i += blockDim.x) dst[i] = p[i];
    p += ns * 6;
  }
}

// words (8 bytes) one packed instance needs
static inline size_t ref_pack_words(const hb_reference& r) {
  size_t w = 8 + (size_t)r.n_events + ((size_t)r.n_events + 2) / 2 + (size_t)r.n_targets * 23;
  for (int c = 0; c < 4; ++c) for (int a = 0; a < 3; ++a) w += (size_t)r.n_segments[c][a] * 6;
  return w;
}
// one instance's packed stream at p (ref_pack_words(r) words)
static inline void ref_pack_one(const hb_reference& r, double* p) {
  RefPackHeader hd;
  memset(&hd, 0, sizeof(hd));
  hd.n_events = r.n_events; hd.n_targets = r.n_targets;
  for (int q = 0; q < 12; ++q) hd.nseg[q] = r.n_segments[q / 3][q % 3];
  memcpy(p, &hd, sizeof(hd)); p += 8;
  memcpy(p, r.event_times, sizeof(double) * r.n_events); p += r.n_events;
  memcpy(p, r.modes, sizeof(int32_t) * (r.n_events + 1)); p += (r.n_events + 2) / 2;
  memcpy(p, r.target_times, sizeof(double) * r.n_targets); p += r.n_targets;
  memcpy(p, r.target_states, sizeof(double) * 22 * r.n_targets); p += 22 * r.n_targets;
  for (int q = 0; q < 12; ++q) { const int ns = r.n_segments[q / 3][q % 3]; memcpy(p, &r.segments[q / 3][q % 3][0][0], sizeof(double) * 6 * ns); p += 6 * ns; }
}
// pack refs[lo, hi) into the pinned staging area dst (offsets first, then the per-instance streams); returns the words used.
// Memory-bound on one core (5.3 MB read from the 17 KB-strided structs and 5.3 MB written per 1024 trot references), inside the caller's
// end-to-end time. Spreading the copies over host threads spawned per call was measured and rejected: on a host with a CPU quota the
// thread start-up costs more than the copies.
static size_t ref_pack(const hb_reference* refs, size_t lo, size_t hi, double* dst) {
  const size_t n = hi - lo;
  long long* offs = reinterpret_cast<long long*>(dst);
  size_t w = n + 1;
  for (size_t i = 0; i < n; ++i) {
    offs[i] = (long long)w;
    ref_pack_one(refs[lo + i], dst + w);
    w += ref_pack_words(refs[lo + i]);
  }
  offs[n] = (long long)w;
  return w;
}

// The rules are written twice and must agree: references_valid checks on the host before a pageable array is packed, and
// reference_gather_pinned_kernel checks a pinned array on the device while it copies it (no host pass over the structs at all).
// Caller-supplied hb_reference structs (host-pointer entry points): counts within the capacities, monotone times, positive segment
// lengths, modes in 0..3. The device expansion indexes with these counts, so a malformed struct is rejected here with HB_EINVAL.
bool references_valid(int B, const hb_reference* refs) {
  for (int i = 0; i < B; ++i) {
    const hb_reference& r = refs[i];
    if (r.n_events < 0 || r.n_events > HB_MAX_EVENTS || r.n_targets < 1 || r.n_targets > HB_MAX_TARGETS) return false;
    for (int k = 0; k <= r.n_events; ++k) if (r.modes[k] < 0 || r.modes[k] > 3) return false;
    for (int k = 0; k < r.n_events; ++k) if (!(r.event_times[k] == r.event_times[k]) || (k > 0 && r.event_times[k] < r.event_times[k - 1])) return false;
    for (int k = 0; k < r.n_targets; ++k) if (!(r.target_times[k] == r.target_times[k]) || (k > 0 && !(r.target_times[k] > r.target_times[k - 1]))) return false;
    for (int c = 0; c < 4; ++c)
      for (int a = 0; a < 3; ++a) {
        const int ns = r.n_segments[c][a];
        if (ns < 0 || ns > HB_MAX_SEGMENTS) return false;
        for (int q = 0; q < ns; ++q) if (!(r.segments[c][a][q][1] > r.segments[c][a][q][0])) return false;
      }
  }
  return true;
}

// The same copy without the host pass: when the caller's hb_reference array is pinned (cudaHostAlloc / cudaHostRegister) the block reads the
// USED entries straight out of host memory through the mapped alias (zero-copy), so no host core packs and only the used bytes cross PCIe.
__global__ void reference_gather_pinned_kernel(int B, const hb_reference* __restrict__ src, hb_reference* refs, unsigned long long* stat) {
  const int inst = blockIdx.x;
  if (inst >= B) return;
  const hb_reference& h = src[inst];
  hb_reference& r = refs[inst];
  __shared__ int cnt[14];
  __shared__ int bad;
  if (threadIdx.x == 0) { bad = 0; cnt[0] = min(max(h.n_events, 0), HB_MAX_EVENTS); if (cnt[0] != h.n_events) bad = 1; }
  __syncthreads();
  if (threadIdx.x == 1) { const int nt = h.n_targets; cnt[1] = min(max(nt, 0), HB_MAX_TARGETS); if (nt < 1 || nt > HB_MAX_TARGETS) bad = 1; }
  if (threadIdx.x >= 2 && threadIdx.x < 14) {
    const int q = threadIdx.x - 2, ns = h.n_segments[q / 3][q % 3];
    cnt[threadIdx.x] = min(max(ns, 0), HB_MAX_SEGMENTS);
    if (ns < 0 || ns > HB_MAX_SEGMENTS) bad = 1;
  }
  __syncthreads();
  const int ne = cnt[0], nt = cnt[1];
  if (threadIdx.x == 0) { r.n_events = ne; r.n_targets = nt; }
  if (threadIdx.x >= 2 && threadIdx.x < 14) { const int q = threadIdx.x - 2; r.n_segments[q / 3][q % 3] = cnt[threadIdx.x]; }
  // the checks of references_valid() ride on the copy: the values are in registers anyway
  bool ok = true;
  for (int i = threadIdx.x; i < ne; i += blockDim.x) {
    const double t = h.event_times[i];
    r.event_times[i] = t;
    if (!(t == t) || (i > 0 && t < h.event_times[i - 1])) ok = false;
  }
  for (int i = threadIdx.x; i <= ne; i += blockDim.x) { const int32_t m = h.modes[i]; r.modes[i] = m; if (m < 0 || m > 3) ok = false; }
  for (int i = threadIdx.x; i < nt; i += blockDim.x) {
    const double t = h.target_times[i];
    r.target_times[i] = t;
    if (!(t == t) || (i > 0 && !(t > h.target_times[i - 1]))) ok = false;
  }
  for (int i = threadIdx.x; i < nt * 22; i += blockDim.x) r.target_states[i / 22][i % 22] = h.target_states[i / 22][i % 22];
  // the twelve (foot, axis) segment lists in one flattened loop: all loads of the block are in flight together (PCIe round trips overlap)
  for (int i = threadIdx.x; i < 12 * HB_MAX_SEGMENTS * 6; i += blockDim.x) {
    const int q = i / (HB_MAX_SEGMENTS * 6), e = i - q * (HB_MAX_SEGMENTS * 6);
    if (e < cnt[2 + q] * 6) {
      const double* sp = &h.segments[q / 3][q % 3][0][0];
      const double v = sp[e];
      (&r.segments[q / 3][q % 3][0][0])[e] = v;
      if (e % 6 == 1 && !(v > sp[e - 1])) ok = false;       // segment end time after its start time
    }
  }
  if (!ok) bad = 1;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (bad) atomicAdd(stat, 1ull);
    int words = 7 + ne + (ne + 2) / 2 + 23 * nt;
    for (int q = 0; q < 12; ++q) words += 6 * cnt[2 + q];
    atomicAdd(stat + 1, (unsigned long long)words);
  }
}

// Time discretisation with event nodes (row S1; ocs2::timeDiscretizationWithEvents as SqpSolver::run calls it): nodes step by dt from the
// initial time; a step that would pass a mode-switch time lands on it instead (the pre-event interval is shortened) and the grid
// re-anchors there; the last node is the final time; nodes closer than dt_min to their predecessor replace it. OCS2's duplicated
// pre- / post-event node pair (identity jump map, no cost, no constraint on it) is collapsed into one node that carries the post-event
// mode. One thread per instance; nn[inst] = number of intervals (<= N, the capacity); status 1 = capacity exhausted (last interval stretched).
__global__ void time_grid_kernel(int B, int N, double dt, double T, const double* t0, const hb_reference* refs, double* tk, int32_t* nn, int32_t* status) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_reference& rf = refs[inst];
  const int nev = min(max(rf.n_events, 0), HB_MAX_EVENTS);
  double* t = tk + (size_t)inst * (N + 1);
  const double ti = t0[inst], tf = ti + T, dt_min = 1e-9;
  int ei = 0;
  while (ei < nev && rf.event_times[ei] <= ti + 1e-9) ++ei;      // switches at (or before) the initial time are in force already
  int n = 0, st = 0;
  double cur = ti;
  t[0] = ti;
  while (cur < tf) {
    double nx = cur + dt;
    if (ei < nev && nx >= rf.event_times[ei]) { nx = rf.event_times[ei]; ++ei; }
    if (nx >= tf) nx = tf;
    if (nx > cur + dt_min || n == 0) {
      if (n == N) { t[N] = tf; st = 1; break; }
      ++n;
    }
    t[n] = nx;
    cur = nx;
  }
  for (int k = n + 1; k <= N; ++k) t[k] = t[n];
  nn[inst] = n;
  if (status) status[inst] = st;
}

// Expansion of the compact reference description onto the node grid (SwitchedModelReferenceManager::modifyReferences
// products evaluated where the solver needs them: TargetTrajectories::getDesiredState, ModeSchedule::modeAtTime,
// SwingTrajectoryPlanner::get{X,Y,Z}{position,velocity}Constraint; CubicSpline.cpp:46-124).
__global__ void reference_expand_kernel(int B, int N, double dt, const double* t0, const hb_reference* refs, double* x_ref, double* swing,
                                        int32_t* mode, const double* tk) {
  const int inst = blockIdx.x;
  const hb_reference& rf = refs[inst];
  // counts are clamped to the capacities of hb_reference: a malformed struct cannot index out of bounds (the host-pointer entry
  // points reject it with HB_EINVAL before it gets here; device-pointer callers own their data)
  const int n_events = min(max(rf.n_events, 0), HB_MAX_EVENTS), n_targets = min(max(rf.n_targets, 1), HB_MAX_TARGETS);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double t = tk ? tk[(size_t)inst * (N + 1) + k] : t0[inst] + k * dt;
    // mode in force on the interval starting at t (post-event mode when t coincides with an event)
    int idx = 0;
    while (idx < n_events && rf.event_times[idx] <= t + 1e-9) ++idx;
    mode[(size_t)inst * (N + 1) + k] = rf.modes[idx];
    // target state: linear interpolation, clamped
    double* xr = x_ref + ((size_t)inst * (N + 1) + k) * NX;
    if (n_targets <= 1 || t <= rf.target_times[0]) { for (int i = 0; i < NX; ++i) xr[i] = rf.target_states[0][i]; }
    else if (t >= rf.target_times[n_targets - 1]) { for (int i = 0; i < NX; ++i) xr[i] = rf.target_states[n_targets - 1][i]; }
    else {
      int s = 0;
      while (s + 2 < n_targets && rf.target_times[s + 1] <= t) ++s;
      const double span = rf.target_times[s + 1] - rf.target_times[s];
      const double al = span > 0.0 ? (t - rf.target_times[s]) / span : 0.0;
      for (int i = 0; i < NX; ++i) xr[i] = (1.0 - al) * rf.target_states[s][i] + al * rf.target_states[s + 1][i];
    }
    // swing references: cubic Hermite segments
    double* sw = swing + ((size_t)inst * (N + 1) + k) * 24;
    for (int c = 0; c < 4; ++c)
      for (int a = 0; a < 3; ++a) {
        const int ns = min(max(rf.n_segments[c][a], 0), HB_MAX_SEGMENTS);
        double pos = 0.0, vel = 0.0;
        if (ns > 0) {
          int s = 0;
          while (s + 1 < ns && t >= rf.segments[c][a][s][1]) ++s;
          const double* sg = rf.segments[c][a][s];
          const double Tr = sg[1] - sg[0], T = Tr > 0.0 ? Tr : 1.0, tn = (t - sg[0]) / T;
          const double dp = sg[4] - sg[2], dvv = sg[5] - sg[3];
          const double c0 = sg[2], c1 = sg[3] * T, c2 = -(3.0 * sg[3] + dvv) * T + 3.0 * dp, c3 = (2.0 * sg[3] + dvv) * T - 2.0 * dp;
          pos = ((c3 * tn + c2) * tn + c1) * tn + c0;
          vel = ((3.0 * c3 * tn + 2.0 * c2) * tn + c1) / T;
        }
        sw[6 * c + a] = pos; sw[6 * c + 3 + a] = vel;
      }
  }
}

// plan_prepare_kernel unpacks t0 / x0 from the plan inputs and evaluates computeFootPos at x0 (the planner's current_feet input).
__global__ void plan_prepare_kernel(int B, const hb_plan_input* in, double* t0, double* x0, double* feet) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_plan_input& p = in[inst];
  for (int i = 0; i < NX; ++i) x0[(size_t)inst * NX + i] = p.x0[i];
  t0[inst] = p.t0;
  contact_positions(p.x0 + 6, feet + (size_t)inst * 12);
}

// Device planner (row N1): the same source as the host planner (csrc/hb_planner.h), four threads per instance (eight instances per 32-thread block). Thread 0 of an
// instance builds the two-sample target in shared memory, thread r plans foot r on it (the feet are independent), thread 0 resamples it,
// then threads 0 and 1 run the IK of the left / right leg on the resampled target, then thread 0 writes the schedule and the targets.
// Same functions as the host planner, so the plan is the same. The targets (2.9 KB each) live in shared memory only: no thread keeps
// a copy on its stack. An instance with a record in targets plans on it instead of its cmd_vel target, where captured (nullable: every
// such instance) has captured[inst] >= 0 (a goal an episode captured). Thread 0 of an instance stages what its plan reads of its record in
// settings (hbplan::PlanSettings: its gait's template and the swing settings; the compiled-in values without a record) in shared memory,
// where the four threads read it. An instance with a record in maps plans on that height map (height maps, hunter_b200.h), which every
// thread reads where it is (a map is 32.8 KB, read at a few points per foot).
__global__ void __launch_bounds__(32) plan_references_coop_kernel(int B, const hb_plan_input* in, const double* feet, double* latest_stance,
                                                                  hb_reference* out, int32_t* status, hbplan::PlanConsts pc,
                                                                  InstanceView<hb_target> targets, const int32_t* captured,
                                                                  InstanceView<hb_planner_settings> settings, InstanceView<hb_terrain> maps) {
  __shared__ hbplan::Target s_tg[8], s_old[8];
  __shared__ hbplan::PlanSettings s_set[8];
  __shared__ int s_rc[8];
  const int g = threadIdx.x >> 2, r = threadIdx.x & 3;
  const int inst = blockIdx.x * 8 + g;
  const bool active = inst < B;
  const hb_terrain* map = active ? maps.of(inst) : nullptr;
  hb_plan_input p;
  hbplan::ModeSchedule ms;
  hb_reference* o = out + (active ? inst : 0);
  double t_lo = 0.0, t_hi = 0.0, tf = 0.0;
  int rc = 0;
  if (r == 0) s_rc[g] = 0;
  __syncwarp();
  if (active) {
    p = in[inst];
    if (feet) for (int i = 0; i < 12; ++i) p.feet_pos[i] = feet[(size_t)inst * 12 + i];
    if (!(p.horizon > 0.0) || !(p.prev_event < p.gait_start) || p.gait < 0 || p.gait > 3) rc = -1;
    tf = p.t0 + p.horizon; t_lo = p.t0 - 1e-9; t_hi = tf + 1e-9;
    if (rc == 0 && r == 0) hbplan::plan_settings(settings.of(inst), p.gait, s_set[g]);
  }
  __syncwarp();
  if (active && rc == 0) {
    if (!hbplan::tile_gait(s_set[g].tmpl, p.prev_event, p.gait_start, p.t0 - p.horizon, tf + p.horizon, ms)) rc = -5;
    if (rc == 0 && r == 0) {
      const hb_target* tg = targets.of(inst);
      if (tg && (!captured || captured[inst] >= 0)) hbplan::target_from(*tg, s_tg[g]);
      else s_tg[g] = hbplan::cmd_vel_to_target(pc, p.cmd_vel, p.t0, p.x0, p.time_to_target, map);
    }
  }
  __syncwarp();
  if (active && rc == 0) {     // rc is the same on the four threads of an instance here
    // phase A: foot r on the two-sample target
    const double body_vel_cmd[6] = {p.cmd_vel[0], p.cmd_vel[1], p.cmd_vel[2], p.cmd_vel[3], 0.0, 0.0};
    hbplan::SwingOut so{o, t_lo, t_hi, false};
    for (int a = 0; a < 3; ++a) o->n_segments[r][a] = 0;
    if (!hbplan::plan_swing(s_set[g], ms, s_tg[g], p.t0, p.feet_pos, body_vel_cmd, latest_stance + (size_t)inst * 12, so, map, r, r + 1) || so.overflow) rc = -5;
  }
  __syncwarp();                // every foot has read the two-sample target before thread 0 resamples it in place
  if (active) {
    if (rc == 0 && r == 0 && p.joint_ik && hbplan::joint_refs_resample(pc, p.t0, tf, s_tg[g], s_old[g]) < 0) rc = -5;
    if (rc != 0) atomicMin(&s_rc[g], rc);
  }
  __syncwarp();
  // phase B: IK per leg on the shared target (segments of every foot are in place after the barrier)
  if (active && s_rc[g] == 0 && p.joint_ik && s_tg[g].n > 2 && r < 2) hbplan::joint_refs_leg(pc, o, r, p.x0, s_tg[g]);
  __syncwarp();
  if (active && r == 0) {
    int frc = s_rc[g];
    if (frc == 0) frc = hbplan::write_schedule_and_targets(ms, s_tg[g], t_lo, t_hi, o);
    if (frc != 0) {
      o->n_events = 0; o->modes[0] = 3; o->n_targets = 1; o->target_times[0] = p.t0;
      for (int i = 0; i < 22; ++i) o->target_states[0][i] = (i < 6) ? 0.0 : p.x0[i];
      for (int c = 0; c < 4; ++c) for (int a = 0; a < 3; ++a) o->n_segments[c][a] = 0;
    }
    if (status) status[inst] = frc;
  }
}
}  // namespace
