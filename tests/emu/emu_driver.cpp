// emu_driver.cpp -- TEST INFRASTRUCTURE (see warp_shim.h).  Runs the frame and stream drivers of the product's
// dexr_kernels.cuh (solve_frame, solve_stream around Solver<G, BW>::solve) on the host: one "warp" = 32 ucontext fibers
// scheduled cooperatively in a single thread, the dynamic shared memory of the CTA = a static buffer, per-group scratch
// laid out like the kernels of dexr.cu lay it out.  What is restated here is only which frames or streams the one emulated
// warp works on: frames are read where they lie in the caller's arrays (the frames kernel stages them in shared memory
// first).  Scratch is poisoned with NaN before every warp call: a value that is read before any lane wrote it must be
// masked by a select.
#include "warp_shim.h"

#include <ucontext.h>

#include <cstdio>
#include <cstdlib>
#include <functional>
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
static std::function<void(int)> lane_fn;

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
static int run_warp(std::function<void(int)> fn) {
  lane_fn = std::move(fn);
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
// Loads the table into the emulated shared memory; returns the byte offset of the scratch, laid out after it.
template <int BW>
int load_table(const dexr_table_t* tb) {
  threadIdx.x = 0; blockDim.x = 1;
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), tb, pass_slot_width<BW>());
  return ((int)sizeof(SharedTable) + 15) / 16 * 16;
}

// One warp call of `fn` on NaN-poisoned scratch.  Returns 0, or a negative code with the message in err.
int run_poisoned(int scratch_off, int scratch_floats, const std::function<void(int)>& fn, const char* what, long long index,
                 char* err, int errlen) {
  if (scratch_off + scratch_floats * 4 > (int)sizeof(dsmem)) {
    snprintf(err, errlen, "emulated shared memory too small");
    return -2;
  }
  uint32_t* sc = reinterpret_cast<uint32_t*>(dsmem + scratch_off);
  for (int i = 0; i < scratch_floats; ++i) sc[i] = 0x7fc00000u;
  if (emu::run_warp(fn) == 0) return 0;
  snprintf(err, errlen, "%s %lld: %s", what, index, emu::errmsg);
  return -1;
}

// dexr_frames_kernel: one frame per group of G lanes, solve_frame writes the outputs.
template <int G, int BW>
int run_frames(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_frames_t& io, long long B, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<BW>(tb);
  const int in_row = io.keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * dm.n_res;
  for (long long base = 0; base < B; base += GPW) {
    auto lane_body = [&](int lane) {
      Solver<G, BW> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * Scratch<G>::kFloats * 4), prm, lane);
      const long long idx = base + lane / G;
      const bool active = idx < B;
      const long long f = active ? idx : base;
      FrameInputs in;
      in.kp = io.keypoints ? io.keypoints + f * in_row : nullptr;
      in.ref = io.keypoints ? nullptr : io.ref_value + f * in_row;
      in.last = io.last_qpos + f * dm.n_var;
      in.fixed = io.fixed_qpos ? io.fixed_qpos + f * dm.n_fixed : nullptr;
      in.projected = io.projected ? io.projected + f * dm.len_proj : nullptr;
      solve_frame(sv, in, io, dm, f, active);
    };
    if (int rc = run_poisoned(scratch_off, GPW * Scratch<G>::kFloats, lane_body, "frame", base, err, errlen)) return rc;
  }
  return 0;
}

// dexr_sequences_kernel with one warp: two streams at a time on 16 lanes, one on 32 lanes or in duo mode (both 16-lane
// groups on the same stream).
template <int G, int BW>
int run_streams(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_sequences_t& io, long long S, int T, bool duo,
                char* err, int errlen) {
  constexpr int GPW = 32 / G;
  duo = duo && G == 16;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<BW>(tb);
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  for (long long base = 0; base < S; base += duo ? 1 : GPW) {
    auto lane_body = [&](int lane) {
      const int gid = lane / G;
      const uint32_t off = (uint32_t)(scratch_off + gid * Scratch<G>::kStreamFloats * 4);
      Solver<G, BW> sv;
      sv.init(tb, dm, off, prm, lane);
      if (duo) sv.duo = gid;
      const long long s = duo ? base : base + gid;
      float* kpbuf = reinterpret_cast<float*>(dsmem + off) + Scratch<G>::kFloats;
      solve_stream(sv, io, dm, prm, S, T, s, s < S, s < S && (!duo || gid == 0), kpbuf, use_filter);
    };
    if (int rc = run_poisoned(scratch_off, GPW * Scratch<G>::kStreamFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// Emulated dexr_solve_frames / dexr_solve_sequences: the library's choice of solver instantiation, with use_arrow in place of
// DEXR_ARROW.  Return 0, or a negative code with a message in err.
extern "C" int emu_solve_frames(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow, const dexr_frames_t* io,
                                long long B, char* err, int errlen) {
  return with_solver(solver_kind(*tb, use_arrow), [&](auto s) {
    return run_frames<decltype(s)::G, decltype(s)::BW>(tb, *prm, *io, B, err, errlen);
  });
}

extern "C" int emu_solve_sequences(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow, const dexr_sequences_t* io,
                                   long long S, long long T, int duo, char* err, int errlen) {
  if (S <= 0 || T <= 0) return 0;
  const dexr_params_t sp = sequence_params(*prm);
  return with_solver(solver_kind(*tb, use_arrow), [&](auto s) {
    return run_streams<decltype(s)::G, decltype(s)::BW>(tb, sp, *io, S, (int)T, duo != 0, err, errlen);
  });
}

extern "C" long long emu_rounds() { return emu::n_rounds_total; }
