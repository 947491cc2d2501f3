// emu_driver.cpp -- TEST INFRASTRUCTURE (see warp_shim.h).  Runs Solver<G, BW>::solve from the product's
// dexr_kernels.cuh on the host: one "warp" = 32 ucontext fibers scheduled cooperatively in a single thread, the dynamic
// shared memory of the CTA = a static buffer, per-group scratch laid out like the frames kernel does (dexr.cu
// launch_frames / dexr_frames_kernel: one frame per group of G lanes, same FrameInputs, same outputs).  Scratch is
// poisoned with NaN before every warp call: a value that is read before any lane wrote it must be masked by a select.
#include "warp_shim.h"

#include <ucontext.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../dex_retargeting_b200/csrc/dexr_kernels.cuh"

emu_dim3 threadIdx{0, 0, 0}, blockDim{1, 1, 1}, blockIdx{0, 0, 0}, gridDim{1, 1, 1};
namespace dexr {
__attribute__((aligned(16))) unsigned char dsmem[256 * 1024];
}

namespace emu {
constexpr int W = 32;
static ucontext_t main_ctx, ctx[W];
static std::vector<char> stacks[W];
static int cur = -1;
static bool finished[W], arrived[W];
static int arr_op[W];
static uint32_t arr_val[W], snap[W];
static void* arr_site[W];
static char errmsg[512];
static long long n_rounds_total = 0;
static void (*lane_fn)(int);

int lane() { return cur; }

__attribute__((noinline)) const uint32_t* rendezvous(int op, uint32_t value) {
  const int me = cur;
  arr_op[me] = op;
  arr_val[me] = value;
  arr_site[me] = __builtin_return_address(0);
  arrived[me] = true;
  swapcontext(&ctx[me], &main_ctx);
  return snap;  // consumed by this fiber before any other fiber runs
}

static void trampoline(int l) {
  lane_fn(l);
  finished[l] = true;
}

// Runs fn(lane) on 32 lanes in lock step.  0 = all lanes returned; -1 = protocol violation (errmsg).
static int run_warp(void (*fn)(int)) {
  lane_fn = fn;
  for (int l = 0; l < W; ++l) {
    finished[l] = arrived[l] = false;
    getcontext(&ctx[l]);
    if (stacks[l].empty()) stacks[l].resize(1 << 20);
    ctx[l].uc_stack.ss_sp = stacks[l].data();
    ctx[l].uc_stack.ss_size = stacks[l].size();
    ctx[l].uc_link = &main_ctx;
    makecontext(&ctx[l], (void (*)())trampoline, 1, l);
  }
  for (;;) {
    for (int l = 0; l < W; ++l)
      if (!finished[l] && !arrived[l]) {
        cur = l;
        swapcontext(&main_ctx, &ctx[l]);
      }
    int nfin = 0, narr = 0;
    for (int l = 0; l < W; ++l) { nfin += finished[l]; narr += arrived[l]; }
    if (nfin == W) return 0;
    if (nfin > 0) {
      snprintf(errmsg, sizeof errmsg, "%d lanes returned while %d wait at a collective (op %d)", nfin, narr, arr_op[0]);
      return -1;
    }
    for (int l = 1; l < W; ++l)
      if (arr_op[l] != arr_op[0] || arr_site[l] != arr_site[0]) {
        snprintf(errmsg, sizeof errmsg, "divergent collectives: lane 0 at op %d site %p, lane %d at op %d site %p", arr_op[0],
                 arr_site[0], l, arr_op[l], arr_site[l]);
        return -1;
      }
    for (int l = 0; l < W; ++l) { snap[l] = arr_val[l]; arrived[l] = false; }
    ++n_rounds_total;
  }
}
}  // namespace emu

using namespace dexr;

namespace {
struct Job {
  const dexr_table_t* tb;
  dexr_params_t prm;
  Dims dm;
  int scratch_off;
  const float *kp, *ref, *last, *fixed;
  uint8_t* projected;
  long long B, base;
  float *qpos_out, *robot_qpos_out, *cost_out, *damping_io;
  int* status_out;
} job;

template <int G, int BW>
void lane_body(int lane) {
  const Job& j = job;
  const int gid = lane / G;
  Solver<G, BW> sv;
  sv.init(j.tb, j.dm, (uint32_t)(j.scratch_off + gid * Scratch<G>::kFloats * 4), j.prm, lane);
  const long long idx = j.base + gid;
  const bool active = idx < j.B;
  const long long f = active ? idx : j.base;
  FrameInputs in;
  in.kp = j.kp ? j.kp + f * 3 * DEXR_NUM_KEYPOINTS : nullptr;
  in.ref = j.kp ? nullptr : j.ref + f * 3 * j.dm.n_res;
  in.last = j.last + f * j.dm.n_var;
  in.fixed = j.fixed ? j.fixed + f * j.dm.n_fixed : nullptr;
  in.projected = j.projected ? j.projected + f * j.dm.len_proj : nullptr;
  sv.lam_carry = j.damping_io ? j.damping_io[f] : 0.f;
  const int status = sv.solve(in, active);
  if (active) {
    if (sv.l == 0 && j.damping_io) j.damping_io[f] = sv.lam_carry;
    if (sv.var >= 0) j.qpos_out[f * j.dm.n_var + sv.var] = sv.x;
    if (j.robot_qpos_out && sv.l < j.dm.dof) j.robot_qpos_out[f * j.dm.dof + sv.l] = sv.q;
    if (sv.l == 0) {
      if (j.status_out) j.status_out[f] = status;
      if (j.cost_out) j.cost_out[f] = sv.F;
    }
  }
}

template <int G, int BW>
int run_all(char* err, int errlen) {
  constexpr int GPW = 32 / G;
  job.scratch_off = ((int)sizeof(SharedTable) + 15) / 16 * 16;
  const int scratch_bytes = GPW * Scratch<G>::kFloats * 4;
  if (job.scratch_off + scratch_bytes > (int)sizeof(dsmem)) { snprintf(err, errlen, "emulated shared memory too small"); return -2; }
  threadIdx.x = 0; blockDim.x = 1;
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), job.tb, pass_slot_width<BW>());
  for (job.base = 0; job.base < job.B; job.base += GPW) {
    uint32_t* sc = reinterpret_cast<uint32_t*>(dsmem + job.scratch_off);
    for (int i = 0; i < scratch_bytes / 4; ++i) sc[i] = 0x7fc00000u;  // NaN poison
    if (emu::run_warp(&lane_body<G, BW>) != 0) {
      snprintf(err, errlen, "frame %lld: %s", job.base, emu::errmsg);
      return -1;
    }
  }
  return 0;
}
}  // namespace

// Same dispatch as dexr_solve_frames (dexr.cu): 16 lanes per frame up to 16 DoF (block mode if the table says so), else 32
// (arrow mode if the table qualifies and use_arrow).  Returns 0, or a negative code with a message in err.
extern "C" int emu_solve_frames(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow, const float* keypoints,
                                const float* ref_value, const float* last_qpos, const float* fixed_qpos, uint8_t* projected,
                                long long B, float* qpos_out, float* robot_qpos_out, int* status_out, float* cost_out, float* damping_io,
                                char* err, int errlen) {
  job = Job{};
  job.tb = tb; job.prm = *prm;
  Dims& d = job.dm;
  d.dof = tb->dof; d.n_var = tb->n_var; d.n_fixed = tb->n_fixed; d.n_links = tb->n_links; d.n_res = tb->n_res; d.loss = tb->loss;
  d.n_rounds = tb->n_rounds; d.has_mimic = tb->has_mimic; d.num_fingers = tb->num_fingers; d.len_proj = tb->len_proj;
  d.len_s1 = tb->len_s1; d.block_width = tb->block_width; d.trunk = tb->arrow > 0 ? tb->arrow - 1 : 0;
  job.kp = keypoints; job.ref = ref_value; job.last = last_qpos; job.fixed = fixed_qpos; job.projected = projected;
  job.B = B; job.qpos_out = qpos_out; job.robot_qpos_out = robot_qpos_out; job.status_out = status_out; job.cost_out = cost_out;
  job.damping_io = damping_io;
  if (tb->dof <= 16) return tb->block_width == 4 ? run_all<16, 4>(err, errlen) : run_all<16, 0>(err, errlen);
  if (tb->arrow > 0 && use_arrow) return run_all<32, -1>(err, errlen);
  return run_all<32, 0>(err, errlen);
}

// ------------------------------------------------------------------------------------------------------------------
// Streams.  The per-stream recurrence of dexr_sequences_kernel (dexr.cu) restated around the same Solver::solve: warm start
// carried in the lane's register (in.last == nullptr), clip, solve, unfiltered solution = next warm start, low-pass filter
// on the full joint vector, DexPilot flags read-modify-written in place.  (The kernel stages each frame's keypoints in
// shared memory first; here solve() reads them where they are.)
namespace {
struct SeqJob {
  dexr_sequences_t io;
  long long S, base;
  int T;
  int duo;  // 16-lane solver: both groups of the warp work on stream `base` (dexr_sequences_kernel with spw == 1)
} sjob;

template <int G, int BW>
void seq_lane_body(int lane) {
  const Job& j = job;
  const SeqJob& q = sjob;
  const int gid = lane / G;
  Solver<G, BW> sv;
  sv.init(j.tb, j.dm, (uint32_t)(j.scratch_off + gid * Scratch<G>::kFloats * 4), j.prm, lane);
  const bool duo = G == 16 && q.duo;
  if (duo) sv.duo = gid;
  const int l = sv.l;
  const bool use_filter = j.prm.lp_alpha >= 0.f && j.prm.lp_alpha <= 1.f;
  const long long s = duo ? q.base : q.base + gid;
  const bool active = s < q.S;
  const bool writes = active && (!duo || gid == 0);
  const long long sc = active ? s : q.S - 1;
  float last = 0.f, fy = 0.f;
  int finit = 0;
  if (active && sv.var >= 0) last = q.io.last_qpos[sc * j.dm.n_var + sv.var];
  if (active && use_filter && l < j.dm.dof) fy = q.io.filter_state[sc * j.dm.dof + l];
  if (active && use_filter) finit = q.io.filter_init[sc];
  sv.lam_carry = (active && q.io.damping_state) ? q.io.damping_state[sc] : 0.f;
  for (int t = 0; t < q.T; ++t) {
    FrameInputs in;
    in.kp = q.io.keypoints + (sc * q.T + t) * 3 * DEXR_NUM_KEYPOINTS;
    in.ref = nullptr;
    in.fixed = j.dm.n_fixed > 0 ? q.io.fixed_qpos + (sc * q.T + t) * j.dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = q.io.projected ? q.io.projected + sc * j.dm.len_proj : nullptr;
    sv.x = last;
    const int status = sv.solve(in, active);
    last = sv.x;
    float out = sv.q;
    if (use_filter) {
      fy = finit ? fmaf(j.prm.lp_alpha, out - fy, fy) : out;
      finit = 1;
      out = fy;
    }
    if (writes) {
      if (l < j.dm.dof) q.io.robot_qpos_out[(sc * q.T + t) * j.dm.dof + l] = out;
      if (l == 0 && q.io.status_out) q.io.status_out[sc * q.T + t] = status;
    }
    __syncwarp();
  }
  if (writes) {
    if (sv.var >= 0) q.io.last_qpos[sc * j.dm.n_var + sv.var] = last;
    if (use_filter && l < j.dm.dof) q.io.filter_state[sc * j.dm.dof + l] = fy;
    if (use_filter && l == 0) q.io.filter_init[sc] = (uint8_t)finit;
    if (q.io.damping_state && l == 0) q.io.damping_state[sc] = sv.lam_carry;
  }
}

template <int G, int BW>
int run_streams(char* err, int errlen) {
  constexpr int GPW = 32 / G;
  job.scratch_off = ((int)sizeof(SharedTable) + 15) / 16 * 16;
  const int scratch_bytes = GPW * Scratch<G>::kFloats * 4;
  threadIdx.x = 0; blockDim.x = 1;
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), job.tb, pass_slot_width<BW>());
  for (sjob.base = 0; sjob.base < sjob.S; sjob.base += (G == 16 && sjob.duo) ? 1 : GPW) {
    uint32_t* sc = reinterpret_cast<uint32_t*>(dsmem + job.scratch_off);
    for (int i = 0; i < scratch_bytes / 4; ++i) sc[i] = 0x7fc00000u;
    if (emu::run_warp(&seq_lane_body<G, BW>) != 0) {
      snprintf(err, errlen, "stream %lld: %s", sjob.base, emu::errmsg);
      return -1;
    }
  }
  return 0;
}
}  // namespace

extern "C" int emu_solve_sequences(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow, const dexr_sequences_t* io,
                                   long long S, long long T, int duo, char* err, int errlen) {
  job = Job{};
  job.tb = tb; job.prm = *prm;
  job.prm.clip_init = 1;  // launch_sequences: SeqRetargeting.retarget always clips the warm start
  Dims& d = job.dm;
  d.dof = tb->dof; d.n_var = tb->n_var; d.n_fixed = tb->n_fixed; d.n_links = tb->n_links; d.n_res = tb->n_res; d.loss = tb->loss;
  d.n_rounds = tb->n_rounds; d.has_mimic = tb->has_mimic; d.num_fingers = tb->num_fingers; d.len_proj = tb->len_proj;
  d.len_s1 = tb->len_s1; d.block_width = tb->block_width; d.trunk = tb->arrow > 0 ? tb->arrow - 1 : 0;
  sjob.io = *io; sjob.S = S; sjob.T = (int)T; sjob.duo = duo;
  if (S <= 0 || T <= 0) return 0;
  if (tb->dof <= 16) return tb->block_width == 4 ? run_streams<16, 4>(err, errlen) : run_streams<16, 0>(err, errlen);
  if (tb->arrow > 0 && use_arrow) return run_streams<32, -1>(err, errlen);
  return run_streams<32, 0>(err, errlen);
}

extern "C" long long emu_rounds() { return emu::n_rounds_total; }
