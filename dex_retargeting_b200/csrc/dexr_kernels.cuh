// dexr_kernels.cuh -- the fused per-frame retargeting solver for sm_90a (H100).
//
// One group of G lanes (G = 16 or 32, so two or one hand-frames per warp) owns one hand-frame.
// Lane c of the group is movable joint c of the robot in pinocchio DoF order.  Everything the
// reference does per frame on the CPU through nlopt + pinocchio + torch
// (optimizer.py:77-102, 146-198, 249-304, 510-575; robot_wrapper.py:82-95;
// kinematics_adaptor.py:102-113 -- paths relative to src/dex_retargeting of the reference repository) happens here
// without leaving the SM:
//   * forward kinematics by pointer jumping over the joint tree (log2(depth) rounds of a 12-float
//     warp shuffle + 3x4 compose); the 3x4 joint placements live in shared memory (one LDS.128 per
//     matrix element triple), the small per-lane constants in registers for the kernel's lifetime;
//   * world-aligned linear Jacobian columns a_c x (p_link - p_c), one column per lane;
//   * the Position / Vector / DexPilot Huber objective, its exact gradient and its exact Hessian:
//     sum_k Jv_k^T (d2 loss/dr2) Jv_k  +  FK curvature  a_i . sum_l (J_lj x dF/dp_l)  +  2 norm_delta I,
//     built by broadcasting Jacobian rows through shared memory;
//   * a bounded Levenberg-Marquardt / Newton iteration: active-set freeze at the box bounds,
//     in-register Cholesky (lane = row) written as a ROLLED loop (rows rotate one column per pivot, so
//     the pivot column is always register 0) with fused forward substitution, shared-memory-transposed
//     back substitution, noise-aware step acceptance in fp32;
//   * block mode (template parameter BW): robots whose fingers are kinematically decoupled (Allegro,
//     LEAP with a palm-fixed origin link) have a block-diagonal Newton system; all blocks are built and
//     factorised side by side, BW pivots instead of dof;
//   * DexPilot hysteresis flags, weights and projected targets (optimizer.py:456-508);
//   * for sequences, SeqRetargeting's clip -> solve -> scatter -> mimic -> low-pass recurrence
//     (seq_retarget.py:112-134, optimizer_utils.py:7-13) carried in registers across time steps.
// Inputs of a batch are staged HBM (or pinned host memory, zero-copy) -> shared memory by a producer warp
// with cp.async.bulk (TMA 1-D) into a two-stage ring guarded by mbarriers; consumer warps claim frames
// from the ring dynamically.
// No tensor cores: n <= 32 unknowns per frame, the work is FP32 issue / latency bound.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dexr.h"

// Experiment switches (compile time; `python -m dex_retargeting_b200.build --variants` builds one library per switch
// next to the default one, selected at run time with DEXR_LIBRARY).  The default build defines none of them.
//   DEXR_EXP_FASTSINCOS  MUFU sine / cosine (__sincosf, abs. error ~5e-7 on [-pi, pi]) instead of sincosf
// Former switches that are the default since round 2:
//   * the short run-time loops of the FK rounds / link placement stay ROLLED (`DEXR_ROLL`): the compiler otherwise unrolls
//     them 3-4x with remainder loops for trip counts of 1-2, and the LM loop body is instruction-fetch bound;
//   * MERGED RESIDUAL PASSES: a residual only touches the joints above its links; residuals that touch disjoint sets of lane
//     slots (block mode: the BW-lane windows; dense mode: 4-lane chunks) are packed into the same pass (greedy, once
//     per CTA: SharedTable::pass_res) and every lane works on the residual of its slot, instead of all lanes walking all
//     n_res residuals.  Allegro / LEAP vector: 1 pass instead of 4; DexPilot on a palm-fixed hand: the wrist -> tip vectors
//     share a pass and disjoint finger pairs share passes (4 instead of 10).  Hands with wrist joints above every finger get
//     no merging (every residual touches the trunk slot).  The terms a lane no longer visits were exact zeros: same sums, up
//     to the sign of zero.  Not used in arrow mode or with mimic joints (one residual per pass there).
//   * the NOISE FLOOR of the objective used by the acceptance test is kNoise |F| PLUS the fp32 resolution of the link
//     positions seen through the loss, 2 ulp x sum_k w_k |p_k|_1 (the Huber slope is at most 1): with link positions of
//     0.5-5 m (free-flying base) F ~ 1e-3 is only resolved to ~2e-8, ten times coarser than kNoise |F|, and a converging
//     Newton step used to be rejected on a noise bump (Shadow position, shipped +-5 m range: 1.5 % of the bench frames
//     ended up to 4e-4 rad from the float64 minimiser; now all within 4e-6).
//   * POSITIVE-DEFINITE FALLBACK: when the factorisation of the exact Hessian fails (the kinematic curvature term makes it
//     indefinite far from the solution), that term is taken back out of the stored Hessian and the trial is repeated at the
//     SAME damping with the positive semi-definite model, instead of multiplying the damping by 10 and refactorising until
//     it dominates (Shadow position bench frames: 6.8 -> 4.5 iterations and 2.2 -> 0.05 extra factorisations per frame).
#define DEXR_ROLL _Pragma("unroll 1")
// Iteration trace: only in the host emulation (tests/emu) when built with -DDEXR_TRACE; expands to nothing in CUDA builds.
#if defined(DEXR_HOST_EMULATION) && defined(DEXR_TRACE)
#include <cstdio>
#define DEXR_TRACE_PRINT(...) do { if (l == 0) { std::printf(__VA_ARGS__); } } while (0)
#else
#define DEXR_TRACE_PRINT(...) do { } while (0)
#endif

namespace dexr {

// The whole dynamic shared memory of a CTA.  Declared once at namespace scope so that every access below is
// a shared-window access with a compile-time offset (LDS/STS [reg + imm]) instead of a generic pointer.
extern __shared__ __align__(16) unsigned char dsmem[];

constexpr int kMaxTrials = 8;
constexpr float kNoise = 5e-7f;      // relative fp32 noise floor of a term-by-term objective difference (a few ulp per term)
constexpr float kLamMin = 1e-7f;
constexpr float kLamDown = 0.1f;
constexpr float kLamUp = 10.0f;
constexpr float kGradNoise = 1e-7f;  // |dF/dx| below this is indistinguishable from 0 in fp32
constexpr float kNearStep = 0.1f;    // accepted step (rad / m) below which the exact radial loss curvature is used
constexpr float kFarResidual = 1e30f; // (round 1 left the kinematic curvature out beyond 0.2 m because it makes the Hessian indefinite far
                                     // from the targets; the positive-definite fallback now handles that case, and on targets out of reach
                                     // the term is what makes the iteration quadratic: 25-60 -> 4-8 iterations)
// Damping schedule beyond "x 0.1 after a verified decrease, x 10 after a rejected step":
//  * a decrease that matches the quadratic model's prediction to within kModelGood relaxes the damping by a second factor
//    kLamDown: the model is as good as it gets, the remaining damping only slows the iteration down (bench frames, mean
//    iterations: Shadow position 4.14 -> 3.96, LEAP DexPilot 3.69 -> 3.53, config-4 streams 4.54 -> 4.12);
//  * a STREAM remembers the damping its last frame needed for its first accepted step and starts the next frame at kCarry
//    times that (never below params.lambda0) -- dexr_frames_t.damping_io / dexr_sequences_t.damping_state.  Stretches of a
//    trajectory where the exact Hessian is nearly singular at the optimum (pinched DexPilot poses) otherwise pay the same
//    two rejected steps at the start of every frame (config-4 streams: rejected steps per frame 1.24 -> 0.66, and the
//    free-running stream follows the oracle's minima more often: 0.77 -> 0.85 of the frames).
constexpr float kModelGood = 0.1f;
constexpr float kCarry = 0.3f;
constexpr float kTrustDecrease = 0.9f;  // a trusted step counts as progress when the gradient max-norm shrank below this factor
// Stop one iteration ahead: the last iteration of a converging frame only confirms that its step is below the tolerance
// (typical steps 5e-2, 4e-3, 1e-5, 2e-7 rad against tol = 1e-5).  When two consecutive first-trial steps contract by
// rho = s_k / s_(k-1) the next one is at most rho s_k as long as the contraction does not get worse (it gets better:
// the damping shrinks and Newton's rate is quadratic), so the frame ends after step k once s_k^2 / s_(k-1) < kStopAhead tol.
constexpr float kStopAhead = 0.5f;
constexpr float kStopAheadRate = 0.02f;  // contraction better than this per step is not extrapolated (a step right after a bound
                                         // was released, or whose max-norm sits in a fast subspace, can look 100x better than the next)

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
template <int G>
__device__ __forceinline__ float gshfl(float v, int src) {
  return __shfl_sync(0xffffffffu, v, src, G);
}
template <int G>
__device__ __forceinline__ int gshfl_i(int v, int src) {
  return __shfl_sync(0xffffffffu, v, src, G);
}
template <int G>
__device__ __forceinline__ float gsum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
  return v;
}
template <int G>
__device__ __forceinline__ float gmax(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o, G));
  return v;
}
template <int G>
__device__ __forceinline__ bool gany(bool p, int lane) {
  unsigned b = __ballot_sync(0xffffffffu, p);
  if (G == 32) return b != 0u;
  return ((b >> (lane & ~(G - 1))) & ((1u << (G & 31)) - 1u)) != 0u;
}
template <int G>
__device__ __forceinline__ unsigned gballot(bool p, int lane) {
  unsigned b = __ballot_sync(0xffffffffu, p);
  if (G == 32) return b;
  return (b >> (lane & ~(G - 1))) & ((1u << (G & 31)) - 1u);
}

template <int N>
struct ChunkTag { static constexpr int value = N; };

// 1 / sqrt(x) for x >= 1e-20 (no denormals, no zero): the bare MUFU.RSQ (rsqrt.approx.ftz, 2^-22 relative) -- rsqrtf() wraps it
// in a denormal rescue of four more instructions, once per Cholesky pivot
__device__ __forceinline__ float fast_rsqrt(float x) {
#ifndef DEXR_HOST_EMULATION
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return 1.0f / sqrtf(x);
#endif
}

// 1 / x for normal positive x: the bare MUFU.RCP (rcp.approx.ftz, 1 ulp) instead of the 8-9 instruction sequences behind
// __fdividef / __frcp_rn; the callers exclude zero and denormal arguments
__device__ __forceinline__ float fast_rcp(float x) {
#ifndef DEXR_HOST_EMULATION
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return 1.0f / x;
#endif
}

__device__ __forceinline__ float huber_val(float d, float beta, float inv_beta) {
  return d < beta ? 0.5f * d * d * inv_beta : d - 0.5f * beta;
}

#ifndef DEXR_HOST_EMULATION  // tests/emu compiles this header for the host: no PTX there (the kernels stay in dexr.cu)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
#endif  // DEXR_HOST_EMULATION

// Problem dimensions: passed as kernel arguments (constant bank) so that every loop bound and branch that
// depends on them is provably warp-uniform for the compiler (no divergence scaffolding around shuffles).
struct Dims {
  int dof, n_var, n_fixed, n_links, n_res, loss, n_rounds, has_mimic, num_fingers, len_proj, len_s1;
  int block_width;  // the table's: 0 = dense Hessian; 4 / 8 = the Hessian is block diagonal over aligned lane windows of this
                    // width (only Solver<16, 4> factorises block by block; every other instantiation treats it as dense)
  int trunk;        // arrow mode only: number of trunk lanes (lanes 0..trunk-1), see Solver
};

inline Dims make_dims(const dexr_table_t& t) {
  Dims d;
  d.dof = t.dof; d.n_var = t.n_var; d.n_fixed = t.n_fixed; d.n_links = t.n_links; d.n_res = t.n_res; d.loss = t.loss;
  d.n_rounds = t.n_rounds; d.has_mimic = t.has_mimic; d.num_fingers = t.num_fingers; d.len_proj = t.len_proj;
  d.len_s1 = t.len_s1;
  d.block_width = t.block_width;
  d.trunk = t.arrow > 0 ? t.arrow - 1 : 0;
  return d;
}

// ------------------------------------------------------------------------------------------------
// uniform (per CTA) slice of the robot table kept in shared memory
// ------------------------------------------------------------------------------------------------
struct SharedTable {
  // per lane, element i of the 3x3 joint placement: (R0[i], RA[i], RB[i], w) with w = p0[i] (i<3), d0[i-3]
  // (3<=i<6), axis[i-6] (6<=i<9); [i][lane] so that a group's LDS.128 is conflict free
  float4 lane_c[9][DEXR_MAX_LANES];
  // links riding on each lane: (offset xyz, slot as int bits; slot -1 = none), `own_rounds` entries per lane
  float4 lane_link[DEXR_MAX_LINKS_PER_LANE][DEXR_MAX_LANES];
  int own_rounds;
  float clip_lo[DEXR_MAX_LANES], clip_hi[DEXR_MAX_LANES];
  int fixed_index[DEXR_MAX_LANES];
  float4 link_off[DEXR_MAX_LINKS];  // xyz, w = parent lane as int bits
  uint32_t link_anc[DEXR_MAX_LINKS];
  int res_task[DEXR_MAX_RES], res_origin[DEXR_MAX_RES], res_ht[DEXR_MAX_RES], res_ho[DEXR_MAX_RES];
  int s2_origin[DEXR_MAX_RES], s2_task[DEXR_MAX_RES];
  int group_count[DEXR_MAX_LANES];
  int group_lane[DEXR_MAX_LANES][DEXR_MAX_GROUP];
  float group_mult[DEXR_MAX_LANES][DEXR_MAX_GROUP];
  // pass_res[r][slot]: the residual the lanes of `slot` work on in pass r, -1 = none (slot = lane / pass_slot_width<BW>() of
  // the Solver instantiation that reads it: BW lanes in block mode, 4 in dense mode -- also for a table with block_width 8,
  // which runs densely because there is no <G, 8> instantiation)
  int pass_res[DEXR_MAX_RES][DEXR_MAX_LANES / 4];
  int n_pass;
};

// Lanes per residual-pass slot of Solver<G, BW>: the schedule in SharedTable::pass_res must be built with the width the
// running instantiation reads it with, not with the table's block_width.
template <int BW>
__host__ __device__ constexpr int pass_slot_width() { return BW > 0 ? BW : 4; }

// slot_width: pass_slot_width<BW>() of the Solver instantiation that runs on this table.  The default, 4, is that width for
// every instantiation there is (<16, 4>, <16, 0>, <32, 0>, and <32, -1>, which does not read the schedule); a table with
// block_width 8 runs densely and gets 4-lane slots too.
__device__ inline void load_shared_table(SharedTable& st, const dexr_table_t* __restrict__ tb, int slot_width = 4) {
  for (int i = threadIdx.x; i < DEXR_MAX_LINKS; i += blockDim.x) {
    st.link_off[i] = make_float4(tb->link_off[i][0], tb->link_off[i][1], tb->link_off[i][2],
                                 __int_as_float(tb->link_parent[i]));
    st.link_anc[i] = tb->link_anc_mask[i];
  }
  for (int i = threadIdx.x; i < DEXR_MAX_RES; i += blockDim.x) {
    st.res_task[i] = tb->res_task[i];
    st.res_origin[i] = tb->res_origin[i];
    st.res_ht[i] = tb->res_human_task[i];
    st.res_ho[i] = tb->res_human_origin[i];
    st.s2_origin[i] = tb->s2_origin[i];
    st.s2_task[i] = tb->s2_task[i];
  }
  for (int i = threadIdx.x; i < DEXR_MAX_LANES; i += blockDim.x) {
    int cnt = 0;
    for (int k = 0; k < tb->n_links; ++k)
      if (tb->link_parent[k] == i && cnt < DEXR_MAX_LINKS_PER_LANE)
        st.lane_link[cnt++][i] = make_float4(tb->link_off[k][0], tb->link_off[k][1], tb->link_off[k][2], __int_as_float(k));
    for (int k = cnt; k < DEXR_MAX_LINKS_PER_LANE; ++k) st.lane_link[k][i] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
    for (int e = 0; e < 9; ++e) {
      const float w = e < 3 ? tb->p0[i][e] : (e < 6 ? tb->d0[i][e - 3] : tb->axis[i][e - 6]);
      st.lane_c[e][i] = make_float4(tb->R0[i][e], tb->RA[i][e], tb->RB[i][e], w);
    }
    st.clip_lo[i] = tb->clip_lo[i];
    st.clip_hi[i] = tb->clip_hi[i];
    st.fixed_index[i] = tb->fixed_index[i];
    st.group_count[i] = tb->group_count[i];
    if (i == 0) {  // most links any single lane carries (1 for every shipped hand)
      int mx = 0;
      for (int c = 0; c < DEXR_MAX_LANES; ++c) {
        int n = 0;
        for (int k = 0; k < tb->n_links; ++k) n += (tb->link_parent[k] == c);
        mx = n > mx ? n : mx;
      }
      st.own_rounds = mx > DEXR_MAX_LINKS_PER_LANE ? DEXR_MAX_LINKS_PER_LANE : mx;
      {
        const int gr = slot_width;  // lanes per slot
        const int nslot = DEXR_MAX_LANES / 4;
        const bool merge = !(tb->block_width == 0 && tb->has_mimic);  // mimic fold: keep one residual per pass
        for (int r = 0; r < DEXR_MAX_RES; ++r)
          for (int sl = 0; sl < nslot; ++sl) st.pass_res[r][sl] = -1;
        int np = 0;
        for (int k = 0; k < tb->n_res; ++k) {
          const uint32_t msk = tb->link_anc_mask[tb->res_task[k]] |
                               (tb->res_origin[k] >= 0 ? tb->link_anc_mask[tb->res_origin[k]] : 0u);
          uint32_t sm = 0u;  // slots this residual touches; one that touches no joint rides in slot 0 (it still counts
          for (int sl = 0; sl < nslot && sl * gr < 32; ++sl)  // for the residual maximum)
            if ((msk >> (sl * gr)) & ((1u << gr) - 1u)) sm |= 1u << sl;
          if (!sm) sm = 1u;
          if (!merge) sm = (1u << nslot) - 1u;
          int r = 0;
          for (;; ++r) {  // first pass whose slots are all free (pass k at the latest: at most k residuals came before)
            bool free_pass = true;
            for (int sl = 0; sl < nslot; ++sl)
              if (((sm >> sl) & 1u) && st.pass_res[r][sl] >= 0) free_pass = false;
            if (free_pass) break;
          }
          for (int sl = 0; sl < nslot; ++sl)
            if ((sm >> sl) & 1u) st.pass_res[r][sl] = k;
          np = r + 1 > np ? r + 1 : np;
        }
        st.n_pass = np;
      }
    }
    for (int f = 0; f < DEXR_MAX_GROUP; ++f) {
      st.group_lane[i][f] = tb->group_lane[i][f];
      st.group_mult[i][f] = tb->group_mult[i][f];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per-group scratch in shared memory (floats)
// ------------------------------------------------------------------------------------------------
template <int G>
struct Scratch {
  static constexpr int NP = G;
  static constexpr int kFr = 0;                                 // [MAX_RES][4] target xyz, weight c_k
  static constexpr int kLp = kFr + DEXR_MAX_RES * 4;            // [2][MAX_LINKS][4] link positions
  static constexpr int kU = kLp + 2 * DEXR_MAX_LINKS * 4;       // jbuf[2][3][NP] (aliased by the 2 Cholesky row buffers) + at: 2 x [NP + NP/4] float4
  static constexpr int kUSize = 16 * NP;
  static constexpr int kHb = kU + kUSize;                       // [NP][NP]   Hessian backup, column per lane
  static constexpr int kLcol = kHb + NP * NP;                   // [NP][NP+1] L^T rows, conflict-free column reads (also mimic-fold temp)
  static constexpr int kFloats = ((kLcol + NP * (NP + 1) + 3) / 4) * 4;
  static constexpr int kStreamFloats = kFloats + 64;  // sequences: followed by the current frame's 63 keypoint floats
};

// ------------------------------------------------------------------------------------------------
// the solver: lane constants + per-frame state in registers
// ------------------------------------------------------------------------------------------------
struct FrameInputs {
  const float* kp;     // 63 floats (keypoints mode) or nullptr
  const float* ref;    // m*3 floats (ref mode) or nullptr
  const float* fixed;  // n_fixed floats or nullptr
  const float* last;   // n_var floats
  uint8_t* projected;  // len_proj flags (global) or nullptr
};

template <int G, int BW = 0>
struct Solver {
  static constexpr int NP = G;
  // BW == 0: dense.  BW > 0: block diagonal over aligned windows of BW lanes.  BW < 0: ARROW -- a trunk (lanes
  // 0..t-1, t <= 8: free-flying base and / or wrist) shared by decoupled fingers (contiguous lane runs of <= 8 joints):
  // H = [F B; B^T W] with F block diagonal.  A finger lane keeps its own finger's row segment (registers 0..7, column
  // fb + j) and its coupling to the trunk (registers 8..15, column j - 8); a trunk lane keeps its row of W in
  // registers 8..15.  Fingers are eliminated side by side (<= 8 pivot steps for all of them), the trunk sees their
  // Schur complement, then the t x t trunk system is factorised: ~13 pivot steps instead of 30 for the Shadow hand
  // on a free-flying base, and half the registers.
  static_assert(BW <= 0 || (BW % 4 == 0 && BW < G), "block width must be a multiple of 4 below the group width");
  static_assert(BW >= 0 || G == 32, "arrow mode is a 32-lane layout");
  static constexpr bool AR = BW < 0;
  static constexpr int HN = (BW == 0) ? G : (AR ? 16 : BW);  // Hessian row segment held per lane
  using SC = Scratch<G>;

  // ---- lane constants kept in registers (the 3x4 joint placement lives in shared memory) ----
  float lo, hi, mmult, moff;
  int jtype, var, msrc;
  uint32_t jump, anc, desc;
  int l;     // lane within group
  int lane;  // lane within warp
  uint32_t sc_off;  // byte offset of this group's scratch inside dsmem
  Dims dm;
  dexr_params_t prm;
  float inv_beta;

  // ---- per-frame state ----
  float x, x0, q, qfix;       // variable value, anchor, full joint value, fixed value
  float p[3], a[3];           // world origin of this joint frame and world axis at the accepted x (the 3x3 world rotation is
                              // transient: it only serves to place the links and to rotate the axis, right after an FK)
  float F;                    // objective at x
  float Fl;                   // this lane's term of F at x (residual l and / or the regulariser of variable l): trial points
                              // are compared term by term, sum_l (v_new - v_old), which resolves differences far below ulp(F)
  float Fnz;                  // sum_k w_k h'(d_k) |p_k|_1 at x: scale of the fp32 position noise in F
  mutable float cost_nz;      // the same for the last cost() call
  mutable float cost_lane;    // this lane's term for the last cost() call
  int cur;                    // which link-position buffer holds the accepted positions
  float lam_carry = 0.f;      // in: damping this frame starts with (<= 0: params.lambda0); out: what the stream's next frame should start with
  int duo = -1;               // 16-lane solver only: -1 = this group owns its frame; 0 / 1 = BOTH groups of the warp work on the same
                              // frame (scarce streams: a stream is latency bound, the second half-warp would idle) and this is
                              // half `duo`: the merged residual passes are dealt alternately to the two halves -- same
                              // instructions, other residuals -- and their partial gradient / Hessian sums are added across the
                              // halves with full-width shuffles.  Everything else runs redundantly in both halves.

  __device__ __forceinline__ static const SharedTable& ST() { return *reinterpret_cast<const SharedTable*>(dsmem); }

  __device__ void init(const dexr_table_t* __restrict__ tb, const Dims& dm_, uint32_t scratch_byte_off,
                       const dexr_params_t& prm_, int lane_) {
    dm = dm_; sc_off = scratch_byte_off; prm = prm_; lane = lane_; l = lane_ & (G - 1);
    inv_beta = 1.0f / prm.huber_delta;
    const int c = l;
    lo = tb->lower[c]; hi = tb->upper[c];
    mmult = tb->mimic_mult[c]; moff = tb->mimic_off[c];
    jtype = tb->jtype[c]; var = tb->var_index[c]; msrc = tb->mimic_src[c];
    jump = tb->jump[c]; anc = tb->anc_mask[c]; desc = tb->desc_mask[c];
  }

  __device__ __forceinline__ float* scf() const { return reinterpret_cast<float*>(dsmem + sc_off); }
  __device__ __forceinline__ float4* fr() const { return reinterpret_cast<float4*>(scf() + SC::kFr); }
  __device__ __forceinline__ float4* lp(int b) const { return reinterpret_cast<float4*>(scf() + SC::kLp) + b * DEXR_MAX_LINKS; }
  __device__ __forceinline__ float* jbuf(int b, int comp) const { return scf() + SC::kU + (b * 3 + comp) * NP; }
  // world axis (a) and torque-like sum (t) of every lane, read back column by column for the kinematic curvature.  One float4
  // per lane and array, with one float4 of padding after every four lanes: the lanes of a group read four different entries at
  // a time (one per 4-lane window in block mode), and a stride of 5 float4 puts those on different banks (the interleaved
  // [lane][a, t] layout of round 1 had every window on the same banks: 23 % of the headline kernel's shared wavefronts)
  // (dense and arrow modes read one entry at a time, broadcast to the whole group: plain index there)
  __device__ __forceinline__ static int at_slot(int i) { return BW > 0 ? i + (i >> 2) : i; }
  __device__ __forceinline__ float4& at_a(int i) const { return reinterpret_cast<float4*>(scf() + SC::kU + 6 * NP)[at_slot(i)]; }
  __device__ __forceinline__ float4& at_t(int i) const { return reinterpret_cast<float4*>(scf() + SC::kU + 6 * NP)[NP + NP / 4 + at_slot(i)]; }
  __device__ __forceinline__ float* lrow() const { return scf() + SC::kU; }
  __device__ __forceinline__ float* hb() const { return scf() + SC::kHb; }
  __device__ __forceinline__ float* lcol() const { return scf() + SC::kLcol; }

  // q of every joint from the variables: target joints copy, fixed joints constant, mimic affine.
  // (optimizer.py:147-151 + kinematics_adaptor.py:102-105)
  __device__ __forceinline__ float compose_q(float xv) const {
    if constexpr (BW != 0) {  // block / arrow tables have neither mimic nor fixed joints (checked on upload): every joint is a
      return var >= 0 ? xv : 0.f;  // variable, and the mimic / fixed-joint state below is dead (register pressure)
    } else {
      const float src = gshfl<G>(xv, msrc >= 0 ? msrc : l);
      return var >= 0 ? xv : (msrc >= 0 ? fmaf(mmult, src, moff) : qfix);
    }
  }

  // Forward kinematics (robot_wrapper.py:82-83 [pinocchio forwardKinematics]) by pointer jumping.
  __device__ __forceinline__ void fk(float qv, float* Ro, float* po) const {
    float s, c;
#ifdef DEXR_EXP_FASTSINCOS
    __sincosf(qv, &s, &c);
#else
    sincosf(qv, &s, &c);
#endif
    const float omc = 1.0f - c;
    const bool rev = jtype == 0;
    float w[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const float4 k = ST().lane_c[i][l];
      Ro[i] = rev ? fmaf(s, k.y, fmaf(omc, k.z, k.x)) : k.x;
      w[i] = k.w;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) po[i] = rev ? w[i] : fmaf(qv, w[3 + i], w[i]);
    const int rounds = dm.n_rounds;
    DEXR_ROLL
    for (int r = 0; r < rounds; ++r) {
      const int src = (jump >> (6 * r)) & 63;
      const bool has = src != 63;
      const int sl = has ? src : l;
      float Rs[9], ps[3];
#pragma unroll
      for (int i = 0; i < 9; ++i) Rs[i] = gshfl<G>(Ro[i], sl);
#pragma unroll
      for (int i = 0; i < 3; ++i) ps[i] = gshfl<G>(po[i], sl);
      if (has) {
        float Rn[9], pn[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
          for (int j = 0; j < 3; ++j)
            Rn[3 * i + j] = fmaf(Rs[3 * i], Ro[j], fmaf(Rs[3 * i + 1], Ro[3 + j], Rs[3 * i + 2] * Ro[6 + j]));
          pn[i] = fmaf(Rs[3 * i], po[0], fmaf(Rs[3 * i + 1], po[1], fmaf(Rs[3 * i + 2], po[2], ps[i])));
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) Ro[i] = Rn[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) po[i] = pn[i];
      }
    }
  }

  // World axis of this lane's joint from its world rotation (the Jacobian column direction, robot_wrapper.py:93-95).
  __device__ __forceinline__ void set_world_axis(const float* Rw) {
    const float ax0 = ST().lane_c[6][l].w, ax1 = ST().lane_c[7][l].w, ax2 = ST().lane_c[8][l].w;
    a[0] = fmaf(Rw[0], ax0, fmaf(Rw[1], ax1, Rw[2] * ax2));
    a[1] = fmaf(Rw[3], ax0, fmaf(Rw[4], ax1, Rw[5] * ax2));
    a[2] = fmaf(Rw[6], ax0, fmaf(Rw[7], ax1, Rw[8] * ax2));
  }

  // Link origins (robot_wrapper.py:85-87 [updateFramePlacement]) -> shared buffer b.  Each lane places the links
  // that ride on its joint (normally one); links fixed to the world are written once per frame (prelude).
  __device__ __forceinline__ void write_links(const float* Rw, const float* pw, int b) const {
    float4* out = lp(b);
    const int rounds = ST().own_rounds;
    DEXR_ROLL
    for (int r = 0; r < rounds; ++r) {
      const float4 o = ST().lane_link[r][l];
      const int slot = __float_as_int(o.w);
      if (slot >= 0)
        out[slot] = make_float4(fmaf(Rw[0], o.x, fmaf(Rw[1], o.y, fmaf(Rw[2], o.z, pw[0]))),
                                fmaf(Rw[3], o.x, fmaf(Rw[4], o.y, fmaf(Rw[5], o.z, pw[1]))),
                                fmaf(Rw[6], o.x, fmaf(Rw[7], o.y, fmaf(Rw[8], o.z, pw[2]))), 0.f);
    }
  }
  __device__ __forceinline__ void write_world_links() const {
    const int L = dm.n_links;
    DEXR_ROLL
    for (int k = l; k < L; k += G) {
      const float4 o = ST().link_off[k];
      if (__float_as_int(o.w) < 0) {
        lp(0)[k] = make_float4(o.x, o.y, o.z, 0.f);
        lp(1)[k] = make_float4(o.x, o.y, o.z, 0.f);
      }
    }
  }

  // Objective L(x) + norm_delta |x - x0|^2 from link buffer b (value part of optimizer.py:162-167,
  // 263-274, 524-541, with the regulariser the reference only puts into the gradient).
  // Sets cost_lane (this lane's term) and cost_nz (group sum of the noise scale); the caller sums what it needs.
  __device__ __forceinline__ void cost(int b, float xv) const {
    float v = 0.f;
    float nz = 0.f;
    const int m = dm.n_res;
    if (l < m) {
      const float4 T = fr()[l];
      const int ti = ST().res_task[l], oi = ST().res_origin[l];
      const float4 pt = lp(b)[ti];
      float rx = pt.x - T.x, ry = pt.y - T.y, rz = pt.z - T.z;
      float ax_ = fabsf(pt.x), ay_ = fabsf(pt.y), az_ = fabsf(pt.z);
      if (oi >= 0) {
        const float4 po = lp(b)[oi];
        rx -= po.x; ry -= po.y; rz -= po.z;
        ax_ += fabsf(po.x); ay_ += fabsf(po.y); az_ += fabsf(po.z);
      }
      const float beta = prm.huber_delta;
      // nz: how far a rounding error of the link positions (relative 2^-24 each) can move this term: |dh/dp| |p|
      if (dm.loss == DEXR_LOSS_POSITION) {
        const float rx_ = fabsf(rx), ry_ = fabsf(ry), rz_ = fabsf(rz);
        v = T.w * (huber_val(rx_, beta, inv_beta) + huber_val(ry_, beta, inv_beta) + huber_val(rz_, beta, inv_beta));
        nz = T.w * fmaf(fminf(rx_ * inv_beta, 1.f), ax_, fmaf(fminf(ry_ * inv_beta, 1.f), ay_, fminf(rz_ * inv_beta, 1.f) * az_));
      } else {
        const float d = sqrtf(fmaf(rx, rx, fmaf(ry, ry, rz * rz)));
        v = T.w * huber_val(d, beta, inv_beta);
        nz = T.w * fminf(d * inv_beta, 1.f) * (ax_ + ay_ + az_);
      }
    }
    if (var >= 0) {
      const float dx = xv - x0;
      v = fmaf(prm.norm_delta * dx, dx, v);
    }
    cost_lane = v;
    cost_nz = gsum<G>(nz);
  }

  // Per-frame targets and weights -> fr[k]; DexPilot flag update (optimizer.py:460-508).
  // Returns false if an input is non finite.
  __device__ __forceinline__ bool prepare_targets(const FrameInputs& in, bool active) {
    const int m = dm.n_res;
    const int loss = dm.loss;
    float tx = 0.f, ty = 0.f, tz = 0.f, w = 0.f;
    if (active && l < m) {
      if (in.kp != nullptr) {
        const int ht = ST().res_ht[l], ho = ST().res_ho[l];
        tx = in.kp[3 * ht]; ty = in.kp[3 * ht + 1]; tz = in.kp[3 * ht + 2];
        if (ho >= 0) { tx -= in.kp[3 * ho]; ty -= in.kp[3 * ho + 1]; tz -= in.kp[3 * ho + 2]; }
        if (prm.preprocess != 0) {
          // Raw detector landmarks (single_hand_detector.py:100-103, 130-158): the map to wrist-centred MANO-convention
          // points is p -> (p - wrist) . [x | n | z] . operator2mano, linear in p, so a vector target only needs the
          // 3x3 part applied to the difference of its two landmarks and a position target to (landmark - wrist).
          // Frame: n = plane normal of {wrist, index base (5), middle base (9)} (the reference takes it from an SVD: the
          // same line up to sign), x = wrist - middle base made orthogonal to n, z = x x n, signs fixed so that z points
          // from the middle base to the index base.  Every lane of the group computes it (uniform loads).
          const float wx = in.kp[0], wy = in.kp[1], wz = in.kp[2];
          if (ho < 0) { tx -= wx; ty -= wy; tz -= wz; }
          const float ax = in.kp[15] - wx, ay = in.kp[16] - wy, az = in.kp[17] - wz;
          const float bx = in.kp[27] - wx, by = in.kp[28] - wy, bz = in.kp[29] - wz;
          float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz_ = ax * by - ay * bx;
          const float nn = rsqrtf(nx * nx + ny * ny + nz_ * nz_);
          nx *= nn; ny *= nn; nz_ *= nn;
          float xx = -bx, xy = -by, xz = -bz;
          const float dn = xx * nx + xy * ny + xz * nz_;
          xx -= dn * nx; xy -= dn * ny; xz -= dn * nz_;
          const float xn_ = rsqrtf(xx * xx + xy * xy + xz * xz);
          xx *= xn_; xy *= xn_; xz *= xn_;
          float zx = xy * nz_ - xz * ny, zy = xz * nx - xx * nz_, zz = xx * ny - xy * nx;
          if (zx * (ax - bx) + zy * (ay - by) + zz * (az - bz) < 0.f) { nx = -nx; ny = -ny; nz_ = -nz_; zx = -zx; zy = -zy; zz = -zz; }
          const float sgn = prm.preprocess == 2 ? -1.f : 1.f;  // operator2mano: right [[0,0,-1],[-1,0,0],[0,1,0]], left mirrors y
          const float u = tx * xx + ty * xy + tz * xz, v = tx * nx + ty * ny + tz * nz_, w_ = tx * zx + ty * zy + tz * zz;
          tx = -sgn * v; ty = sgn * w_; tz = -u;
        }
      } else {
        tx = in.ref[3 * l]; ty = in.ref[3 * l + 1]; tz = in.ref[3 * l + 2];
      }
    }
    bool finite = isfinite(tx) && isfinite(ty) && isfinite(tz);
    if (loss == DEXR_LOSS_POSITION) {
      w = 1.0f / (3.0f * m);
    } else if (loss == DEXR_LOSS_VECTOR) {
      tx *= prm.scaling; ty *= prm.scaling; tz *= prm.scaling;
      w = 1.0f / m;
    } else {
      const int len_proj = dm.len_proj, len_s1 = dm.len_s1;
      const float dist = sqrtf(fmaf(tx, tx, fmaf(ty, ty, tz * tz)));
      int flag = 0;
      if (l < len_s1) {
        flag = (active && in.projected != nullptr) ? in.projected[l] : 0;
        if (dist < prm.project_dist) flag = 1;
        if (dist > prm.escape_dist) flag = 0;
      }
      const int k2 = l - len_s1;
      const bool is_s2 = (l >= len_s1) && (l < len_proj);
      const int so = is_s2 ? ST().s2_origin[k2] : 0, sk = is_s2 ? ST().s2_task[k2] : 0;
      const int fo = gshfl_i<G>(flag, so), fk_ = gshfl_i<G>(flag, sk);
      if (is_s2) flag = (fo && fk_ && dist <= 0.03f) ? 1 : 0;
      float weight;
      if (l < len_proj) {
        weight = flag ? (l < len_s1 ? 200.0f : 400.0f) : 1.0f;
        if (flag) {
          const float sc_ = (l < len_s1 ? prm.eta1 : prm.eta2) / (dist + 1e-6f);
          tx *= sc_; ty *= sc_; tz *= sc_;
        } else {
          tx *= prm.scaling; ty *= prm.scaling; tz *= prm.scaling;
        }
        if (active && in.projected != nullptr) in.projected[l] = (uint8_t)flag;
      } else {
        weight = (float)(len_proj + dm.num_fingers);
        tx *= prm.scaling; ty *= prm.scaling; tz *= prm.scaling;
      }
      w = weight / m;
    }
    if (l < m) fr()[l] = make_float4(tx, ty, tz, w);
    return !gany<G>(!finite, lane);
  }

  // ---------------------------------------------------------------------------------------------
  // One frame.  Returns status word.  On exit x (var lanes) and q (all lanes) hold the solution.
  // ---------------------------------------------------------------------------------------------
  __device__ __forceinline__ int solve(const FrameInputs& in, bool active) {
    const int dof = dm.dof;
    const float nd = prm.norm_delta;
    const float beta = prm.huber_delta;
    int status = 0;

    // ---- prelude: warm start, anchor, fixed joints (optimizer.py:138-141, seq_retarget.py:115-121)
    float xin = 0.f;
    if (in.last == nullptr) xin = var >= 0 ? x : 0.f;  // sequences: previous solution kept in registers
    else if (active && var >= 0) xin = in.last[var];
    if (prm.clip_init && var >= 0) xin = fminf(fmaxf(xin, ST().clip_lo[l]), ST().clip_hi[l]);
    x0 = xin;
    x = fminf(fmaxf(xin, lo), hi);
    const int fixedi = BW != 0 ? -1 : ST().fixed_index[l];
    qfix = (active && fixedi >= 0) ? in.fixed[fixedi] : 0.f;
    bool finite = isfinite(xin) && isfinite(qfix);
    const bool ok_in = prepare_targets(in, active);
    finite = !gany<G>(!finite, lane) && ok_in;
    __syncwarp();
    if (!finite) {
      status |= DEXR_STATUS_NONFINITE;
      x = x0;
      if (!isfinite(x)) x = 0.f;
      if (!isfinite(qfix)) qfix = 0.f;
      active = false;
    }
    q = compose_q(x);
    {
      float R[9];
      fk(q, R, p);
      cur = 0;
      write_world_links();
      write_links(R, p, cur);
      set_world_axis(R);
    }
    __syncwarp();
    cost(cur, x);
    Fnz = cost_nz;
    Fl = cost_lane;
    F = gsum<G>(Fl);

    float lam = lam_carry > 0.f ? lam_carry : prm.lambda0;  // (kCarry)
    lam_carry = prm.lambda0;
    int iters = 0, rejects = 0;
    bool done = !active;
    // Curvature model (group-uniform): `exact` = use the true second derivative of the norm-Huber loss
    // (radial direction has zero curvature beyond beta); otherwise its quadratic majoriser 1/d * I, which
    // is positive semi-definite and globally safer.  Optimistic start, demoted after a large or failed step.
    bool exact = true;
    // A tiny accepted step ends the frame -- unless some variable is held at a bound: then the gradient is
    // re-evaluated once more, and the frame ends only if the same set stays active (KKT on the bounds).
    bool recheck = false;
    int rechecks = 0;
    unsigned last_fmask = 0u;
    // Steps whose predicted decrease is below what fp32 resolves in F are taken on trust; whether they were any good is read
    // off the GRADIENT one iteration later (it is computed directly, not by differencing F, and resolves far below the noise
    // of F).  A smaller gradient max-norm keeps the step and relaxes the damping like a verified decrease would.  A gradient
    // that did not shrink REVERTS the step: the next trial is forced back to the previous point (x_prev; the forward
    // kinematics and the objective terms are re-evaluated through the ordinary trial code) and the damping goes up, so the
    // gradient norm is monotone over trusted steps -- no cycling between an overshooting and a damped step (seen on targets
    // far out of reach), no creeping at a damping collected early (round 1: 583 of 614 400 DexPilot stream frames ran into
    // max_iters).  Two reverts in a row mean the KKT residual sits at its fp32 floor: the frame ends at the best point.
    float gn_prev = 0.f, x_prev = 0.f;
    float s_prev = 0.f;  // the previous iteration's accepted step when that was a first-trial Newton step, else 0
    bool trust_prev = false;
    int stall = 0;

    // ---- arrow mode: this lane's finger window (see the Solver comment); loop invariant ----
    int ar_t = 0, ar_fb = 0, ar_fw = 0, ar_maxw = 0, ar_fo = 0;
    bool ar_trunk = false;
    if constexpr (AR) {
      ar_t = dm.trunk;
      ar_trunk = l < ar_t;
      const uint32_t tmask = (1u << ar_t) - 1u;
      const bool fin = !ar_trunk && l < dof;
      ar_fb = fin ? __ffs((anc | (1u << l)) & ~tmask) - 1 : 0;  // the finger's first joint: lowest non-trunk ancestor
      const unsigned bases = gballot<G>(fin && ar_fb == l, lane);
      ar_fo = fin ? 8 * (1 + __popc(bases & ((1u << ar_fb) - 1u))) : 0;  // this finger's slot in the small row buffers
      const uint32_t dmask = (uint32_t)gshfl_i<G>((int)desc, ar_fb) | (1u << ar_fb);
      ar_fw = fin ? (32 - __clz(dmask)) - ar_fb : 0;
      ar_maxw = (int)gmax<G>((float)ar_fw);
    }

    while (gany<32>(!done, lane)) {
      // ======================= gradient + exact Hessian at x ===========================
      float H[HN];
#pragma unroll
      for (int i = 0; i < HN; ++i) H[i] = 0.f;
      float g = 0.f, t0 = 0.f, t1 = 0.f, t2 = 0.f;
      const bool rev = jtype == 0;
      const int m = dm.n_res;
      const int loss = dm.loss;
      // Block mode: when the kinematic chains are decoupled (every residual touches one finger and the fingers
      // share no movable ancestor) the Hessian is block diagonal.  Each lane then keeps only its own block's row
      // segment -- register H[j] holds column cb + j -- and all blocks are factorised at the same time: bw
      // pivots instead of dof.  Dense mode is the same code with bw = NP and cb = 0.
      constexpr bool dense = BW == 0;
      const int bw = dense ? dof : BW;
      const int cb = dense ? 0 : (l & ~(BW - 1));
      const float4* lpc = lp(cur);
      float rmax = 0.f;
      constexpr bool merged = !AR;  // merged residual passes (arrow mode keeps one residual per pass)
      int trips = m;
      if constexpr (merged) trips = ST().n_pass;
      const bool two_halves = merged && G == 16 && duo >= 0;
      const int n_pass = trips;
      if (two_halves) trips = (trips + 1) >> 1;
      for (int kk = 0; kk < trips; ++kk) {
        int k = kk;
        bool on = true;  // merged mode: false on the lanes of a slot that has no residual in this pass
        if constexpr (merged) {
          const int kq = two_halves ? 2 * kk + duo : kk;       // this half's pass
          const int kw = ST().pass_res[kq < n_pass ? kq : 0][l / pass_slot_width<BW>()];
          on = kq < n_pass && kw >= 0;
          k = on ? kw : 0;
        }
        const int ti = ST().res_task[k], oi = ST().res_origin[k];
        const float4 T = fr()[k];
        const float4 pt = lpc[ti];
        const uint32_t mt = on ? ST().link_anc[ti] : 0u;
        float rx = pt.x - T.x, ry = pt.y - T.y, rz = pt.z - T.z;
        float j0 = 0.f, j1 = 0.f, j2 = 0.f;
        if ((mt >> l) & 1u) {
          if (rev) {
            const float dx = pt.x - p[0], dy = pt.y - p[1], dz = pt.z - p[2];
            j0 = a[1] * dz - a[2] * dy; j1 = a[2] * dx - a[0] * dz; j2 = a[0] * dy - a[1] * dx;
          } else { j0 = a[0]; j1 = a[1]; j2 = a[2]; }
        }
        uint32_t mo = 0u;
        if (oi >= 0) {
          const float4 po = lpc[oi];
          mo = on ? ST().link_anc[oi] : 0u;
          rx -= po.x; ry -= po.y; rz -= po.z;
          if ((mo >> l) & 1u) {
            if (rev) {
              const float dx = po.x - p[0], dy = po.y - p[1], dz = po.z - p[2];
              j0 -= a[1] * dz - a[2] * dy; j1 -= a[2] * dx - a[0] * dz; j2 -= a[0] * dy - a[1] * dx;
            } else { j0 -= a[0]; j1 -= a[1]; j2 -= a[2]; }
          }
        }
        // loss derivatives wrt the residual block (uniform across lanes)
        float gx, gy, gz, y0, y1, y2;
        if (loss == DEXR_LOSS_POSITION) {
          // per-coordinate Huber: exact curvature is 0 beyond beta; the majoriser 1/max(|r|, beta) is
          // used throughout (identical inside the quadratic zone)
          const float ax_ = fabsf(rx), ay_ = fabsf(ry), az_ = fabsf(rz);
          rmax = on ? fmaxf(rmax, fmaxf(ax_, fmaxf(ay_, az_))) : rmax;
          // 1/beta exactly inside the quadratic zone; beyond it the fast reciprocal (<= 2 ulp) is plenty: it only
          // scales a unit-magnitude gradient component and the majoriser curvature
          const float wx = ax_ < beta ? inv_beta : fast_rcp(ax_);
          const float wy = ay_ < beta ? inv_beta : fast_rcp(ay_);
          const float wz = az_ < beta ? inv_beta : fast_rcp(az_);
          gx = T.w * rx * wx; gy = T.w * ry * wy; gz = T.w * rz * wz;
          y0 = T.w * wx * j0; y1 = T.w * wy * j1; y2 = T.w * wz * j2;
        } else {
          const float d = sqrtf(fmaf(rx, rx, fmaf(ry, ry, rz * rz)));
          rmax = on ? fmaxf(rmax, d) : rmax;
          const bool quad = d < beta;
          const float invd = d > 1e-30f ? fast_rcp(d) : 0.f;
          const float ux = rx * invd, uy = ry * invd, uz = rz * invd;
          const float hp = quad ? d * inv_beta : 1.0f;
          gx = T.w * hp * ux; gy = T.w * hp * uy; gz = T.w * hp * uz;
          const float s_iso = T.w * (quad ? inv_beta : invd);
          const float s_rad = (quad || !exact) ? 0.f : T.w * invd;
          const float uj = s_rad * fmaf(ux, j0, fmaf(uy, j1, uz * j2));
          y0 = fmaf(s_iso, j0, -uj * ux); y1 = fmaf(s_iso, j1, -uj * uy); y2 = fmaf(s_iso, j2, -uj * uz);
        }
        g = fmaf(j0, gx, fmaf(j1, gy, fmaf(j2, gz, g)));
        t0 += j1 * gz - j2 * gy; t1 += j2 * gx - j0 * gz; t2 += j0 * gy - j1 * gx;
        const int b = kk & 1;
        jbuf(b, 0)[l] = j0; jbuf(b, 1)[l] = j1; jbuf(b, 2)[l] = j2;
        __syncwarp();
        const uint32_t cols = mt | mo;
        if constexpr (AR) {
          // trunk columns (aligned float4 chunks at lanes 0.. and 4..) into registers 8..15
#pragma unroll
          for (int blk = 0; blk < 2; ++blk) {
            if (4 * blk < ar_t) {
              const float4 c0 = *reinterpret_cast<const float4*>(jbuf(b, 0) + 4 * blk);
              const float4 c1 = *reinterpret_cast<const float4*>(jbuf(b, 1) + 4 * blk);
              const float4 c2 = *reinterpret_cast<const float4*>(jbuf(b, 2) + 4 * blk);
              H[8 + 4 * blk + 0] = fmaf(c0.x, y0, fmaf(c1.x, y1, fmaf(c2.x, y2, H[8 + 4 * blk + 0])));
              H[8 + 4 * blk + 1] = fmaf(c0.y, y0, fmaf(c1.y, y1, fmaf(c2.y, y2, H[8 + 4 * blk + 1])));
              H[8 + 4 * blk + 2] = fmaf(c0.z, y0, fmaf(c1.z, y1, fmaf(c2.z, y2, H[8 + 4 * blk + 2])));
              H[8 + 4 * blk + 3] = fmaf(c0.w, y0, fmaf(c1.w, y1, fmaf(c2.w, y2, H[8 + 4 * blk + 3])));
            }
          }
          // own finger's columns fb .. fb + fw - 1 (unaligned: scalar loads, one address per finger) into registers 0..7
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (j < ar_maxw) {
              // (the clamp costs two instructions per column; without it ptxas keeps more addresses live and spills 24 bytes
              // more in the 128-register arrow kernel, which then runs slower)
              const int cj = ar_fb + j < NP ? ar_fb + j : NP - 1;
              const float v = fmaf(jbuf(b, 0)[cj], y0, fmaf(jbuf(b, 1)[cj], y1, jbuf(b, 2)[cj] * y2));
              H[j] += j < ar_fw ? v : 0.f;
            }
          }
        }
#pragma unroll
        for (int blk = 0; blk < (AR ? 0 : HN / 4); ++blk) {
          if (4 * blk < bw && (!dense || ((cols >> (4 * blk)) & 0xFu))) {
            const int c4 = cb + 4 * blk;  // first of the four columns this chunk accumulates
            const float4 c0 = *reinterpret_cast<const float4*>(jbuf(b, 0) + c4);
            const float4 c1 = *reinterpret_cast<const float4*>(jbuf(b, 1) + c4);
            const float4 c2 = *reinterpret_cast<const float4*>(jbuf(b, 2) + c4);
            H[4 * blk + 0] = fmaf(c0.x, y0, fmaf(c1.x, y1, fmaf(c2.x, y2, H[4 * blk + 0])));
            H[4 * blk + 1] = fmaf(c0.y, y0, fmaf(c1.y, y1, fmaf(c2.y, y2, H[4 * blk + 1])));
            H[4 * blk + 2] = fmaf(c0.z, y0, fmaf(c1.z, y1, fmaf(c2.z, y2, H[4 * blk + 2])));
            H[4 * blk + 3] = fmaf(c0.w, y0, fmaf(c1.w, y1, fmaf(c2.w, y2, H[4 * blk + 3])));
          }
        }
      }
      if constexpr (merged) rmax = gmax<G>(rmax);  // every window saw only its own residuals
      if constexpr (merged && G == 16) {
        if (two_halves) {  // add the other half's passes (warp-uniform branch: both halves of a warp are in this mode or neither)
          rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, 16));
          g += __shfl_xor_sync(0xffffffffu, g, 16);
          t0 += __shfl_xor_sync(0xffffffffu, t0, 16);
          t1 += __shfl_xor_sync(0xffffffffu, t1, 16);
          t2 += __shfl_xor_sync(0xffffffffu, t2, 16);
#pragma unroll
          for (int i = 0; i < HN; ++i) H[i] += __shfl_xor_sync(0xffffffffu, H[i], 16);
        }
      }
      if constexpr (AR) {  // the aligned trunk chunks also swept columns ar_t..7 (finger lanes): not trunk couplings
#pragma unroll
        for (int c = 0; c < 8; ++c) H[8 + c] = c < ar_t ? H[8 + c] : 0.f;
      }
      // ---- FK curvature: S[i][c] = a_i . t_c (i ancestor-or-self of c), symmetric otherwise ----
      {
        const float ar0 = rev ? a[0] : 0.f, ar1 = rev ? a[1] : 0.f, ar2 = rev ? a[2] : 0.f;
        const bool curv_on = rmax < kFarResidual;  // far from the targets the term is large and indefinite
        at_a(l) = make_float4(ar0, ar1, ar2, 0.f);
        at_t(l) = make_float4(t0, t1, t2, 0.f);
        __syncwarp();
#pragma unroll
        for (int j = 0; j < HN; ++j) {
          if (AR ? (j < 8 ? j < ar_maxw : j - 8 < ar_t) : j < bw) {
            // the joint this register column stands for (arrow mode: clamped; columns a lane does not own add 0 below)
            const int i = AR ? (j < 8 ? (ar_fb + j < NP ? ar_fb + j : NP - 1) : j - 8) : cb + j;
            const float4 ai = at_a(i);
            const float4 ti_ = at_t(i);
            const bool up = (anc >> i) & 1u;
            const bool dn = (desc >> i) & 1u;
            const float vu = fmaf(ai.x, t0, fmaf(ai.y, t1, ai.z * t2));
            const float vd = fmaf(ar0, ti_.x, fmaf(ar1, ti_.y, ar2 * ti_.z));
            const bool mine = !AR || (j < 8 ? j < ar_fw : true);
            H[j] += (curv_on && mine) ? (up ? vu : (dn ? vd : 0.f)) : 0.f;
          }
        }
      }
      // the kinematic curvature is part of H and can be taken out again (not after the mimic fold has mixed it in)
      bool curv_in = rmax < kFarResidual && !(BW == 0 && dm.has_mimic);
      // ---- mimic fold: H_x = M^T H_q M, g_x = M^T g_q (kinematics_adaptor.py:107-113) ----
      if constexpr (BW == 0) if (dm.has_mimic) {
        const float ml = var >= 0 ? 1.0f : (msrc >= 0 ? mmult : 0.f);
        float* hbuf = hb();
        __syncwarp();
#pragma unroll
        for (int i = 0; i < NP; ++i) hbuf[i * NP + l] = ml * H[i];
        __syncwarp();
#pragma unroll
        for (int i = 0; i < NP; ++i) H[i] = 0.f;
        const int gcount = ST().group_count[l];
        for (int f = 0; f < DEXR_MAX_GROUP; ++f) {
          if (var >= 0 && f < gcount) {
            const int cl = ST().group_lane[l][f];
#pragma unroll
            for (int i = 0; i < NP; ++i) H[i] += hbuf[i * NP + cl];
          }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < HN; ++i) hbuf[i * NP + l] = H[i];
        __syncwarp();
        // row fold through shared memory (runtime loop: keeps the code small; only mimic robots get here)
        float* hrow = lcol();  // NP x NP temporary: the transposed-factor area is idle during the Hessian build
        for (int s = 0; s < dof; ++s) {
          float acc = 0.f;
          const int cnt = ST().group_count[s];
          for (int f = 0; f < cnt; ++f) acc = fmaf(ST().group_mult[s][f], hbuf[ST().group_lane[s][f] * NP + l], acc);
          hrow[s * NP + l] = acc;
        }
#pragma unroll
        for (int s = 0; s < NP; ++s) H[s] = (s < dof) ? hrow[s * NP + l] : 0.f;
        float gx_ = 0.f;
#pragma unroll
        for (int f = 0; f < DEXR_MAX_GROUP; ++f) {
          const bool v = var >= 0 && f < gcount;
          const float gv = gshfl<G>(g, v ? ST().group_lane[l][f] : l);
          if (v) gx_ = fmaf(ST().group_mult[l][f], gv, gx_);
        }
        g = gx_;
        __syncwarp();
      }
      // ---- regulariser, active set (box bounds), freeze ----
      const bool isvar = var >= 0;
      g = isvar ? fmaf(2.0f * nd, x - x0, g) : 0.f;
      // a variable sitting on a bound stays active unless the gradient points inward by more than fp32 noise
      const bool act = isvar && ((x <= lo && g > -kGradNoise) || (x >= hi && g < kGradNoise));
      const bool free_ = isvar && !act;
      const unsigned fmask = gballot<G>(free_, lane);
      const bool any_act = gany<G>(act, lane);
      if (recheck && (fmask == last_fmask || ++rechecks >= 3)) done = true;
      recheck = false;
      last_fmask = fmask;
      // Frozen variables (active bounds, fixed / mimic lanes) get identity rows and columns.  The common case
      // -- every lane below dof is a free variable -- skips this pass entirely (warp-uniform branch); lanes
      // at or above dof have all-zero rows and are never pivots (the factorisation stops at dof).
      if (gany<32>(l < dof && !free_, lane)) {
#pragma unroll
        for (int j = 0; j < HN; ++j) {
          // the column register j stands for (arrow mode: -1 where this lane owns none)
          const int cj = AR ? (j < 8 ? (j < ar_fw ? ar_fb + j : -1) : (j - 8 < ar_t ? j - 8 : -1)) : cb + j;
          const bool keep = free_ && cj >= 0 && ((fmask >> (cj & 31)) & 1u);
          float v = keep ? H[j] : 0.f;
          if (cj == l && !free_ && (!AR || ar_trunk == (j >= 8))) v = 1.0f;
          H[j] = v;
        }
      }
      if (!free_) g = 0.f;
      const float gn = gmax<G>(fabsf(g));
      bool revert = false;
      if (trust_prev && !done) {
        if (gn < gn_prev) {
          if (gn < kTrustDecrease * gn_prev) lam = fmaxf(lam * kLamDown, kLamMin);
          stall = 0;
        } else {
          revert = true;
          ++stall;
        }
      }
      DEXR_TRACE_PRINT("  it %2d gn %.3e gn_prev %.3e trust_prev %d stall %d revert %d lam %.1e\n", iters, gn, gn_prev, (int)trust_prev, stall, (int)revert, lam);
      float* hbuf = hb();
#pragma unroll
      for (int i = 0; i < HN; ++i) hbuf[i * NP + l] = H[i];
      // own diagonal entry (register index = lane id is not addressable: read it back from the column store);
      // the regulariser 2*norm_delta enters on the diagonal at pivot time together with the damping
      const float reg2 = free_ ? 2.0f * nd : 0.f;
      const int dj = AR ? (ar_trunk ? 8 + l : l - ar_fb) : l - cb;  // register holding this lane's diagonal entry
      float hd = free_ ? hbuf[dj * NP + l] + reg2 : 1.0f;
      float D = fabsf(hd) + 1e-6f;
      // ======================= damped Newton trials ====================================
      bool accepted = done;
      float acc_step = 0.f;
      float Rn[9], pn[3];
      for (int trial = 0; trial < kMaxTrials; ++trial) {
        if (!gany<32>(!accepted, lane)) break;
        if (trial > 0) {
#pragma unroll
          for (int i = 0; i < HN; ++i) H[i] = hbuf[i * NP + l];
        }
        float y = -g;
        float myinv = 1.0f;
        bool bad = false;
        float* Lr = lrow();   // two NP-float row buffers, alternating per pivot
        float* Lc = lcol();
        __syncwarp();
        // Cholesky, lane = row, as a ROLLED loop: after pivot k every lane shifts its row one column to the
        // left (fused into the update FMA), so the pivot column is always register H[0] and the loop body is
        // the same code for every k -- 16-32x less code than the unrolled form (instruction-cache bound
        // otherwise), same FMA count thanks to the chunk guard.
        if constexpr (AR) {
          // ================= arrow factorisation: fingers side by side, Schur complement, trunk =================
          // ONE loop body serves both elimination passes (pass 0: every finger at once, pass 1: the trunk, whose rows
          // are moved into the rotating window first) and one body both back-substitution passes: the code of an LM
          // iteration has to stay inside the 32 KB L1.5 instruction cache (DESIGN.md section 3.5).
          // Scratch (all inside regions that are idle here): rowb = two alternating sets of per-finger row segments
          // (8 floats per finger slot, slot 0 = trunk), tbuf = per-finger broadcast of the pivot's scaled trunk
          // coupling, M = [lane][12] finger lanes' L_TF column + forward-substituted rhs (upper half of the backup
          // area, which arrow mode does not use).
          float* rowb = Lr;            // [2][64]
          float* tbuf = Lr + 128;      // [64]
          float* M = hb() + 16 * NP;   // [NP][12]
          const bool fin = !ar_trunk && l < dof;
#pragma unroll 1
          for (int pass = 0; pass < 2; ++pass) {
            const bool mine = pass == 0 ? fin : ar_trunk;           // lanes that are rows of this pass
            const int fbx = pass == 0 ? ar_fb : 0, fox = pass == 0 ? ar_fo : 0;
            const int fwx = pass == 0 ? ar_fw : (ar_trunk ? ar_t : 0);
            const int steps = pass == 0 ? ar_maxw : ar_t, lc0 = pass * 8;
            // step s eliminates row fbx + s of every block of the pass at once
#pragma unroll 1
            for (int s_ = 0; s_ < steps; ++s_) {
              const int pk = fbx + s_;
              const bool act = mine && s_ < fwx;
              float hk = H[0];
              if (act && pk == l) hk += fmaf(lam, D, reg2);
              const float dkk = gshfl<G>(hk, act ? pk : l);
              bad = bad || (act && !(dkk > 1e-20f));
              const float inv = act ? fast_rsqrt(fmaxf(dkk, 1e-20f)) : 1.0f;
              const float lik = hk * inv;                            // L[l][pk] for l >= pk
              const float yk = gshfl<G>(y, act ? pk : l) * inv;      // forward substitution fused
              const bool piv = act && l == pk, below = act && l > pk;
              if (piv) { myinv = inv; y = yk; }
              if (pass == 0 && piv) {                                 // the pivot's coupling to the trunk: L_TF[c][pk], final
#pragma unroll
                for (int c = 0; c < 8; ++c) H[8 + c] *= inv;
                *reinterpret_cast<float4*>(tbuf + fox) = make_float4(H[8], H[9], H[10], H[11]);
                *reinterpret_cast<float4*>(tbuf + fox + 4) = make_float4(H[12], H[13], H[14], H[15]);
              }
              if (below) y = fmaf(-lik, yk, y);
              float* row = rowb + (s_ & 1) * 64 + fox;
              if (below) row[l - pk - 1] = lik;                       // entry j of the segment = L[pk+1+j][pk]
              Lc[(lc0 + s_) * (NP + 1) + l] = (act && l >= pk) ? lik : 0.f;  // transposed copy for the back substitution
              __syncwarp();
              if (gany<32>(below, lane)) {
                const int live = fwx - s_ - 1;                        // columns right of the pivot inside the block
                const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 r0 = *reinterpret_cast<const float4*>(row);
                const float4 r1 = *reinterpret_cast<const float4*>(row + 4);
                const float ml = below ? -lik : 0.f;
                // rotate the window one column to the left (stale segment entries beyond `live` masked out)
                H[0] = fmaf(ml, 0 < live ? r0.x : 0.f, H[1]);
                H[1] = fmaf(ml, 1 < live ? r0.y : 0.f, H[2]);
                H[2] = fmaf(ml, 2 < live ? r0.z : 0.f, H[3]);
                H[3] = fmaf(ml, 3 < live ? r0.w : 0.f, H[4]);
                H[4] = fmaf(ml, 4 < live ? r1.x : 0.f, H[5]);
                H[5] = fmaf(ml, 5 < live ? r1.y : 0.f, H[6]);
                H[6] = fmaf(ml, 6 < live ? r1.z : 0.f, H[7]);
                H[7] = 0.f;
                if (pass == 0) {  // trunk coupling of the rows below the pivot (finished rows keep their final L_TF: ml = 0)
                  const float4 v0 = below ? *reinterpret_cast<const float4*>(tbuf + fox) : z4;      // (a slot nobody wrote
                  const float4 v1 = below ? *reinterpret_cast<const float4*>(tbuf + fox + 4) : z4;  //  may hold NaN: select)
                  H[8] = fmaf(ml, v0.x, H[8]);   H[9] = fmaf(ml, v0.y, H[9]);
                  H[10] = fmaf(ml, v0.z, H[10]); H[11] = fmaf(ml, v0.w, H[11]);
                  H[12] = fmaf(ml, v1.x, H[12]); H[13] = fmaf(ml, v1.y, H[13]);
                  H[14] = fmaf(ml, v1.z, H[14]); H[15] = fmaf(ml, v1.w, H[15]);
                }
              }
              __syncwarp();
            }
            if (pass == 0) {
              // ---- Schur complement: W -= L_TF L_TF^T, rhs_T -= L_TF y_F; every lane takes a quarter of the finger
              // rows; then the trunk rows move into the rotating window for pass 1
              M[l * 12 + 8] = fin ? y : 0.f;
              *reinterpret_cast<float4*>(M + l * 12) = fin ? make_float4(H[8], H[9], H[10], H[11]) : make_float4(0.f, 0.f, 0.f, 0.f);
              *reinterpret_cast<float4*>(M + l * 12 + 4) = fin ? make_float4(H[12], H[13], H[14], H[15]) : make_float4(0.f, 0.f, 0.f, 0.f);
              __syncwarp();
              const int c = l & 7, qd = l >> 3;
              float acc[9];
#pragma unroll
              for (int d = 0; d < 9; ++d) acc[d] = 0.f;
              for (int i = ar_t + qd; i < dof; i += 4) {
                const float mc = M[i * 12 + c];
                const float4 m0 = *reinterpret_cast<const float4*>(M + i * 12);
                const float4 m1 = *reinterpret_cast<const float4*>(M + i * 12 + 4);
                acc[0] = fmaf(mc, m0.x, acc[0]); acc[1] = fmaf(mc, m0.y, acc[1]);
                acc[2] = fmaf(mc, m0.z, acc[2]); acc[3] = fmaf(mc, m0.w, acc[3]);
                acc[4] = fmaf(mc, m1.x, acc[4]); acc[5] = fmaf(mc, m1.y, acc[5]);
                acc[6] = fmaf(mc, m1.z, acc[6]); acc[7] = fmaf(mc, m1.w, acc[7]);
                acc[8] = fmaf(mc, M[i * 12 + 8], acc[8]);
              }
#pragma unroll
              for (int d = 0; d < 9; ++d) {
                acc[d] += __shfl_xor_sync(0xffffffffu, acc[d], 8);
                acc[d] += __shfl_xor_sync(0xffffffffu, acc[d], 16);
              }
              if (ar_trunk) {  // lane l < t <= 8: c == l
#pragma unroll
                for (int d = 0; d < 8; ++d) H[d] = H[8 + d] - acc[d];
                y -= acc[8];
              }
            }
          }
          // ---- back substitution: trunk, then the fingers with the trunk solution folded into their rhs ----
#pragma unroll 1
          for (int pass = 1; pass >= 0; --pass) {
            const bool mine = pass == 0 ? fin : ar_trunk;
            const int fbx = pass == 0 ? ar_fb : 0;
            const int fwx = pass == 0 ? ar_fw : (ar_trunk ? ar_t : 0);
            const int steps = pass == 0 ? ar_maxw : ar_t, lc0 = pass * 8;
            if (pass == 0) {
              const float4 m0 = *reinterpret_cast<const float4*>(M + l * 12);
              const float4 m1 = *reinterpret_cast<const float4*>(M + l * 12 + 4);
              float corr = 0.f;
              corr = fmaf(m0.x, gshfl<G>(y, 0), corr); corr = fmaf(m0.y, gshfl<G>(y, 1), corr);
              corr = fmaf(m0.z, gshfl<G>(y, 2), corr); corr = fmaf(m0.w, gshfl<G>(y, 3), corr);
              corr = fmaf(m1.x, gshfl<G>(y, 4), corr); corr = fmaf(m1.y, gshfl<G>(y, 5), corr);
              corr = fmaf(m1.z, gshfl<G>(y, 6), corr); corr = fmaf(m1.w, gshfl<G>(y, 7), corr);
              if (fin) y -= corr;  // entries beyond t are zero in M (H[8 + c] stays 0 for c >= t)
            }
#pragma unroll 1
            for (int s_ = steps - 1; s_ >= 0; --s_) {
              const int pk = fbx + s_;
              const bool act = mine && s_ < fwx;
              const float xk = gshfl<G>(y * myinv, act ? pk : l);
              if (act && l == pk) y = xk;
              if (act && l < pk) y = fmaf(-Lc[(lc0 + l - fbx) * (NP + 1) + pk], xk, y);
            }
          }
        }
        if constexpr (!AR) {
          // One pivot step, with the number of 4-column chunks of the rotating window it updates fixed at compile time.  The
          // window shrinks by one column per pivot, so the steps are run in PHASES of decreasing chunk count (HN = 16: 4, 3,
          // 2, 1 chunks while more than 12, 8, 4, 0 columns are live) instead of predicating all HN / 4 chunks off one by
          // one: half of the FFMA / LDS.128 issue slots of a 16 x 16 factorisation went into predicated-off instructions.
          constexpr int kMask = dense ? NP - 1 : BW - 1;
          const float shift = fmaf(lam, D, reg2);               // damping + regulariser, added to the pivot at pivot time
          int k = 0;
          auto pivot_steps = [&](auto chunks_tag, int stop_live) {
            constexpr int NC = decltype(chunks_tag)::value;
            for (; k < bw && bw - k - 1 > stop_live; ++k) {
              const int pk = cb + k;  // pivot lane (of this lane's block)
              float hk = H[0];
              if (pk == l) hk += shift;
              const float dkk = gshfl<G>(hk, pk);
              bad = bad || !(dkk > 1e-20f);
              const float inv = fast_rsqrt(fmaxf(dkk, 1e-20f));
              const float lik = hk * inv;                       // L[l][k] (meaningful for l >= k)
              const float yk = gshfl<G>(y, pk) * inv;           // forward substitution fused
              if (l == pk) { myinv = inv; y = yk; }
              if (l > pk) y = fmaf(-lik, yk, y);
              float* row = Lr + (k & 1) * NP + cb;              // two NP-float row buffers, alternating per pivot
              row[(l - pk - 1) & kMask] = lik;                  // entry j of the row = L[pk+1+j][pk]
              Lc[k * (NP + 1) + l] = lik;                       // transposed copy for the back substitution
              __syncwarp();
              const int live = bw - k - 1;                      // columns right of the pivot (inside the block)
#pragma unroll
              for (int j = 0; j < 4 * NC; j += 4) {
                if (j + 4 < 4 * NC || j < live) {               // (only the last chunk of a phase can be entirely dead)
                  const float4 r = *reinterpret_cast<const float4*>(row + j);
                  H[j + 0] = fmaf(-lik, r.x, H[j + 1]);
                  if (j + 2 < HN) H[j + 1] = fmaf(-lik, r.y, H[j + 2]);
                  if (j + 3 < HN) H[j + 2] = fmaf(-lik, r.z, H[j + 3]);
                  if (j + 4 < HN) H[j + 3] = fmaf(-lik, r.w, H[j + 4]);
                }
              }
            }
          };
          if constexpr (HN == 32) {
            pivot_steps(ChunkTag<8>{}, 24); pivot_steps(ChunkTag<6>{}, 16); pivot_steps(ChunkTag<4>{}, 8); pivot_steps(ChunkTag<2>{}, -1);
          } else if constexpr (HN == 16) {
            pivot_steps(ChunkTag<4>{}, 12); pivot_steps(ChunkTag<3>{}, 8); pivot_steps(ChunkTag<2>{}, 4); pivot_steps(ChunkTag<1>{}, -1);
          } else if constexpr (HN == 8) {
            pivot_steps(ChunkTag<2>{}, 4); pivot_steps(ChunkTag<1>{}, -1);
          } else {
            pivot_steps(ChunkTag<HN / 4>{}, -1);
          }
        }
        // back substitution: L^T delta = y (column oriented, transposed copy read conflict free)
        for (int k = (AR ? 0 : bw) - 1; k >= 0; --k) {
          const int pk = cb + k;
          const float xk = gshfl<G>(y * myinv, pk);
          if (l == pk) y = xk;
          if (l < pk) y = fmaf(-Lc[(l - cb) * (NP + 1) + pk], xk, y);
        }
        bad = gany<G>(bad || !isfinite(y), lane) && !revert;  // a reverting group ignores this factorisation
        bool dropped = false;  // this group took the kinematic curvature out in this trial: retry at the same damping
        {
          const bool drop = bad && !accepted && curv_in;
          if (gany<32>(drop, lane)) {
            const float4 a_self = at_a(l);          // (rev ? a : 0), t of this lane, as stored when H was built
            const float4 t_self = at_t(l);
#pragma unroll
            for (int j = 0; j < HN; ++j) {
              if (AR ? (j < 8 ? j < ar_maxw : j - 8 < ar_t) : j < bw) {
                const int i = AR ? (j < 8 ? (ar_fb + j < NP ? ar_fb + j : NP - 1) : j - 8) : cb + j;
                const float4 ai = at_a(i);
                const float4 ti_ = at_t(i);
                const bool up = (anc >> i) & 1u;
                const bool dn = (desc >> i) & 1u;
                const float vu = fmaf(ai.x, t_self.x, fmaf(ai.y, t_self.y, ai.z * t_self.z));
                const float vd = fmaf(a_self.x, ti_.x, fmaf(a_self.y, ti_.y, a_self.z * ti_.z));
                const bool mine = !AR || (j < 8 ? j < ar_fw : true);
                const float v = mine ? (up ? vu : (dn ? vd : 0.f)) : 0.f;
                // same column bookkeeping as the freeze pass: frozen rows / columns stay zero (identity)
                const int cj = AR ? (j < 8 ? (j < ar_fw ? ar_fb + j : -1) : (j - 8 < ar_t ? j - 8 : -1)) : cb + j;
                const bool keep = free_ && cj >= 0 && ((fmask >> (cj & 31)) & 1u);
                if (drop && keep) hbuf[j * NP + l] -= v;
              }
            }
            if (drop) {
              curv_in = false;
              dropped = true;
              hd = free_ ? hbuf[dj * NP + l] + reg2 : 1.0f;
              D = fabsf(hd) + 1e-6f;
            }
          }
        }
        if (!gany<32>(!accepted && !bad, lane)) {  // no pending group has a usable step: no FK needed
          if (!accepted && !dropped) { lam *= kLamUp; ++rejects; }
          continue;
        }
        float xn = free_ ? fminf(fmaxf(x + y, lo), hi) : x;
        if (bad) xn = x;
        if (revert) xn = x_prev;  // (every lane: the variable set that was free during the reverted step may differ)
        const float dx = xn - x;
        const float step = gmax<G>(fabsf(dx));
        const float pred = 0.5f * gsum<G>(dx * fmaf(lam * D, dx, -g));
        const float qn = compose_q(xn);
        fk(qn, Rn, pn);
        write_links(Rn, pn, cur ^ 1);
        __syncwarp();
        cost(cur ^ 1, xn);
        // F(xn) - F(x) summed term by term: every lane differences its own residual / regulariser term (nearby numbers: the
        // subtraction is exact), so the result carries the rounding of the terms -- a few ulp of each -- and of the link
        // positions behind them, not ulp(F)
        const float dF = gsum<G>(cost_lane - Fl);
        const float Fn = F + dF;  // (a few ulp of drift per accepted step; F only scales the noise floor and is reported)
        const float fnoise = fmaf(kNoise, fabsf(F), 2.4e-7f * fmaxf(Fnz, cost_nz));
        // a step taken on trust must at least not raise F by more than its noise
        const bool ok = revert || (!bad && isfinite(Fn) && (dF <= 0.f || ((step < prm.tol || pred < fnoise) && dF <= fnoise)));
        // the damping is relaxed after a decrease that fp32 can resolve: one beyond the worst-case rounding bound, or one that
        // agrees with the quadratic model's prediction to within a half (rounding noise that large would not track it)
        const bool verified = !revert && (dF < -fnoise || (dF < 0.f && fabsf(dF + pred) <= 0.5f * pred));
        DEXR_TRACE_PRINT("  it %2d trial %d lam %.1e exact %d step %.3e pred %.3e F %.9e Fn %.9e dF %.2e noise %.1e bad %d ok %d ver %d fmask %x\n", iters,
                         trial, lam, (int)exact, step, pred, F, Fn, dF, fnoise, (int)bad, (int)ok, (int)verified, fmask);
        if (!accepted) {
          if (ok) {
            x_prev = x;
            x = xn; q = qn; F = Fn;
            Fnz = cost_nz;
            Fl = cost_lane;
            set_world_axis(Rn);
#pragma unroll
            for (int i = 0; i < 3; ++i) p[i] = pn[i];
            cur ^= 1;
            // (see kStopAhead; not with active bounds, extra damping or the majoriser model in play)
            const bool ahead = exact && !any_act && trial == 0 && !revert && lam <= prm.lambda0 &&
                               step * fmaxf(step, kStopAheadRate * s_prev) < kStopAhead * prm.tol * s_prev;
            s_prev = (trial == 0 && !revert) ? step : 0.f;
            if (iters == 0 && !revert) lam_carry = fmaxf(prm.lambda0, kCarry * lam);
            if (verified) lam = fmaxf(lam * kLamDown, kLamMin);
            if (verified && fabsf(dF + pred) <= kModelGood * pred) lam = fmaxf(lam * kLamDown, kLamMin);  // (kModelGood)
            // fnoise is a worst-case bound (every rounding error with the same sign); a decrease beyond an eighth of it is
            // already unlikely to be noise: such a step is kept whatever the next gradient says (it just does not relax
            // the damping).  Only steps whose effect on F is truly unresolved are put to the gradient test.
            trust_prev = !verified && !revert && !(dF < -0.125f * fnoise);
            if (verified) stall = 0;
            gn_prev = gn;
            accepted = true;
            acc_step = step;
            if (revert) {  // back at the previous point: more damping, or the end when this is the second revert in a row
              lam *= kLamUp;
              ++rejects;
              if (stall >= 2) { done = true; status |= DEXR_STATUS_NOISEFLOOR; }
              revert = false;
            } else if (step < prm.tol || ahead) {
              if (any_act) recheck = true;
              else done = true;
            }
          } else {
            if (!dropped)
            {
              lam *= kLamUp;
              ++rejects;
            }
          }
        }
        __syncwarp();
      }
      if (!done) {
        if (!accepted) {
          if (exact) lam = prm.lambda0;  // retry this point with the majoriser model
          else done = true;              // no descent direction left at fp32 resolution
        }
        exact = accepted && acc_step < kNearStep;
        ++iters;
        if (iters >= prm.max_iters && !done) { done = true; status |= DEXR_STATUS_MAXITER; }
      }
    }
    status |= (iters & 0xffff) | ((rejects > 127 ? 127 : rejects) << 16);
    return status;
  }
};

// ------------------------------------------------------------------------------------------------
// which Solver instantiation runs a table
// ------------------------------------------------------------------------------------------------
// The values index per-kind settings (DEXR_FRAMES_WARPS) and order the kinds from fastest to slowest.
enum SolverKind {
  kBlock16 = 0,  // <16, 4>: decoupled 4-joint fingers, block-diagonal Hessian
  kDense16 = 1,  // <16, 0>
  kArrow32 = 2,  // <32, -1>: trunk + decoupled fingers, arrow Hessian
  kDense32 = 3,  // <32, 0>
};

// use_arrow = false runs arrow-qualified tables on the dense 32-lane solver.
inline SolverKind solver_kind(const dexr_table_t& t, bool use_arrow) {
  if (t.dof <= 16) return t.block_width == 4 ? kBlock16 : kDense16;
  return (t.arrow > 0 && use_arrow) ? kArrow32 : kDense32;
}

inline int kind_lanes(int kind) { return kind <= kDense16 ? 16 : 32; }

template <int G_, int BW_>
struct SolverTag {
  static constexpr int G = G_, BW = BW_;
};

// f(SolverTag<G, BW>{}) for the instantiation of `kind`.
template <class F>
auto with_solver(SolverKind kind, F&& f) {
  switch (kind) {
    case kBlock16: return f(SolverTag<16, 4>{});
    case kDense16: return f(SolverTag<16, 0>{});
    case kArrow32: return f(SolverTag<32, -1>{});
    default: return f(SolverTag<32, 0>{});
  }
}

// ------------------------------------------------------------------------------------------------
// frame and stream drivers of the kernels (dexr.cu), also run by the host emulation (tests/emu)
// ------------------------------------------------------------------------------------------------
// One frame of a batch: solve from the frame's carried damping, then write its outputs.  `dm` is the kernel argument's, not
// sv.dm: read from the constant bank, it keeps the register allocation of the frames kernels.
template <int G, int BW>
__device__ __forceinline__ void solve_frame(Solver<G, BW>& sv, const FrameInputs& in, const dexr_frames_t& io, const Dims& dm,
                                            long long f, bool active) {
  sv.lam_carry = io.damping_io ? io.damping_io[f] : 0.f;  // (every lane of the group reads the frame's word)
  const int status = sv.solve(in, active);
  if (active) {
    if (sv.var >= 0) io.qpos_out[f * dm.n_var + sv.var] = sv.x;
    if (io.robot_qpos_out && sv.l < dm.dof) io.robot_qpos_out[f * dm.dof + sv.l] = sv.q;
    if (sv.l == 0) {
      if (io.status_out) io.status_out[f] = status;
      if (io.cost_out) io.cost_out[f] = sv.F;
      if (io.damping_io) io.damping_io[f] = sv.lam_carry;
    }
  }
}

// SeqRetargeting.retarget always clips the warm start (seq_retarget.py:118-120).
inline dexr_params_t sequence_params(dexr_params_t p) {
  p.clip_init = 1;
  return p;
}

// One stream s of S: its `steps` frames in order (seq_retarget.py:112-134), warm start and filter carried in registers.  The
// frame's keypoints are staged in `kpbuf` (63 floats of shared memory), the next frame's are prefetched into registers
// meanwhile.  Every group of a warp walks the time loop (warp-wide shuffles inside solve); a group that is not `active` runs
// it on stream S - 1, and only a group that `writes` stores results and state.  `use_filter`: prm.lp_alpha in [0, 1].
// dm, prm, S and steps are the kernel argument's and `use_filter` is computed once per thread: taken by value here, or
// recomputed per stream, they change the register allocation of the sequences kernels.
template <int G, int BW>
__device__ __forceinline__ void solve_stream(Solver<G, BW>& sv, const dexr_sequences_t& io, const Dims& dm,
                                             const dexr_params_t& prm, const long long& S, const int& steps, long long s,
                                             bool active, bool writes, float* kpbuf, bool use_filter) {
  constexpr int KPL = (3 * DEXR_NUM_KEYPOINTS + G - 1) / G;  // keypoint floats per lane
  const int l = sv.l;
  const long long sc = active ? s : S - 1;
  float last = 0.f, fy = 0.f;
  int finit = 0;
  if (active && sv.var >= 0) last = io.last_qpos[sc * dm.n_var + sv.var];
  if (active && use_filter && l < dm.dof) fy = io.filter_state[sc * dm.dof + l];
  if (active && use_filter) finit = io.filter_init[sc];
  sv.lam_carry = (active && io.damping_state) ? io.damping_state[sc] : 0.f;  // then carried by solve() from frame to frame
  const float* kp_stream = io.keypoints + sc * steps * (3 * DEXR_NUM_KEYPOINTS);
  float pre[KPL];
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    const int e = l + j * G;
    pre[j] = (e < 3 * DEXR_NUM_KEYPOINTS) ? kp_stream[e] : 0.f;
  }
  for (int t = 0; t < steps; ++t) {
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int e = l + j * G;
      if (e < 3 * DEXR_NUM_KEYPOINTS) kpbuf[e] = pre[j];
    }
    if (t + 1 < steps) {
      const float* nxt = kp_stream + (long long)(t + 1) * (3 * DEXR_NUM_KEYPOINTS);
#pragma unroll
      for (int j = 0; j < KPL; ++j) {
        const int e = l + j * G;
        pre[j] = (e < 3 * DEXR_NUM_KEYPOINTS) ? nxt[e] : 0.f;
      }
    }
    __syncwarp();
    FrameInputs in;
    in.kp = kpbuf;
    in.ref = nullptr;
    in.fixed = dm.n_fixed > 0 ? io.fixed_qpos + (sc * steps + t) * dm.n_fixed : nullptr;
    in.last = nullptr;  // warm start comes from the register `x` (previous solution)
    in.projected = io.projected ? io.projected + sc * dm.len_proj : nullptr;
    sv.x = last;
    const int status = sv.solve(in, active);
    last = sv.x;  // unfiltered solution is the next warm start (seq_retarget.py:124)
    float out = sv.q;
    if (use_filter) {  // optimizer_utils.py:7-13
      fy = finit ? fmaf(prm.lp_alpha, out - fy, fy) : out;
      finit = 1;
      out = fy;
    }
    if (writes) {
      if (l < dm.dof) io.robot_qpos_out[(sc * steps + t) * dm.dof + l] = out;
      if (l == 0 && io.status_out) io.status_out[sc * steps + t] = status;
    }
    __syncwarp();
  }
  if (writes) {
    if (sv.var >= 0) io.last_qpos[sc * dm.n_var + sv.var] = last;
    if (use_filter && l < dm.dof) io.filter_state[sc * dm.dof + l] = fy;
    if (use_filter && l == 0) io.filter_init[sc] = (uint8_t)finit;
    if (io.damping_state && l == 0) io.damping_state[sc] = sv.lam_carry;
  }
}

// ------------------------------------------------------------------------------------------------
// objective evaluation (dexr_eval_objective): value and gradient at a given point, no solve
// ------------------------------------------------------------------------------------------------
// The evaluation runs on the dense Solver of the table's lane count.  Block and arrow tables have neither mimic nor fixed
// joints, so the dense compose_q is exact for them, and with no Hessian to build their instantiations have nothing to add.
inline int eval_lanes(const dexr_table_t& t) { return t.dof <= 16 ? 16 : 32; }

// An evaluating group only uses the targets and the link positions of its scratch (Scratch<G>::kFr, kLp).
template <int G>
__host__ __device__ constexpr int eval_scratch_floats() { return Scratch<G>::kU; }

// The argument checks of dexr_eval_objective that read the robot's table: nullptr, or what is wrong.  Host code, so that the
// host emulation rejects the same arguments with the same messages.
inline const char* eval_io_error(const dexr_table_t& t, const dexr_eval_t& io, const dexr_params_t& prm) {
  if (!io.qpos) return "qpos is required";
  if ((io.keypoints != nullptr) == (io.ref_value != nullptr)) return "exactly one of keypoints / ref_value must be given";
  if (prm.preprocess != 0 && !io.keypoints) return "preprocess needs raw keypoints, not ref_value";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  return nullptr;
}

// One frame: the objective at x = qpos[f] as given (no clipping), anchored at last_qpos[f] (or x: no regulariser).  The targets
// and DexPilot flags are prepared by the same prepare_targets a solve runs.  Writes L(x), L(x) + norm_delta |x - x0|^2 (a
// fresh sum: solve() carries its F from step to step, so the two differ by a few ulp per accepted iteration) and the gradient
// of the latter.  `dm` is the kernel argument's (constant bank), as in solve_frame.
template <int G>
__device__ __forceinline__ void evaluate_frame(Solver<G, 0>& sv, const FrameInputs& in, const dexr_eval_t& io, const Dims& dm,
                                               long long f, bool active) {
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l;
  const bool isvar = sv.var >= 0;
  float x = 0.f, x0 = 0.f;
  if (active && isvar) {
    x = io.qpos[f * dm.n_var + sv.var];
    x0 = io.last_qpos ? io.last_qpos[f * dm.n_var + sv.var] : x;
  }
  const int fixedi = st.fixed_index[l];
  sv.qfix = (active && fixedi >= 0) ? in.fixed[fixedi] : 0.f;
  sv.x = x;
  sv.prepare_targets(in, active);
  __syncwarp();
  sv.q = sv.compose_q(x);
  {
    float R[9];
    sv.fk(sv.q, R, sv.p);
    sv.write_world_links();
    sv.write_links(R, sv.p, 0);
    sv.set_world_axis(R);
  }
  __syncwarp();
  sv.x0 = x;  // the regulariser term of every lane is exactly 0 (NaN for a non-finite x): L(x)
  sv.cost(0, x);
  const float loss = gsum<G>(sv.cost_lane);
  sv.x0 = x0;
  sv.cost(0, x);
  const float cost = gsum<G>(sv.cost_lane);

  float g = 0.f;
  if (io.grad_out) {
    // dL/dq of this lane's joint: over the residuals, the loss derivative (the formulas of solve(): per-coordinate Huber slope,
    // h'(d) r / d with 0 at d = 0 as torch's norm backward) dotted with this lane's Jacobian column of task minus origin link.
    // One residual per pass on every lane: solve()'s merged passes and its Hessian are of no use here.
    const float beta = sv.prm.huber_delta, inv_beta = sv.inv_beta;
    const bool rev = sv.jtype == 0;
    const float4* lpc = sv.lp(0);
    for (int k = 0; k < dm.n_res; ++k) {
      const int ti = st.res_task[k], oi = st.res_origin[k];
      const float4 T = sv.fr()[k];
      const float4 pt = lpc[ti];
      float rx = pt.x - T.x, ry = pt.y - T.y, rz = pt.z - T.z;
      float j0 = 0.f, j1 = 0.f, j2 = 0.f;
      if ((st.link_anc[ti] >> l) & 1u) {
        if (rev) {
          const float dx = pt.x - sv.p[0], dy = pt.y - sv.p[1], dz = pt.z - sv.p[2];
          j0 = sv.a[1] * dz - sv.a[2] * dy; j1 = sv.a[2] * dx - sv.a[0] * dz; j2 = sv.a[0] * dy - sv.a[1] * dx;
        } else { j0 = sv.a[0]; j1 = sv.a[1]; j2 = sv.a[2]; }
      }
      if (oi >= 0) {
        const float4 po = lpc[oi];
        rx -= po.x; ry -= po.y; rz -= po.z;
        if ((st.link_anc[oi] >> l) & 1u) {
          if (rev) {
            const float dx = po.x - sv.p[0], dy = po.y - sv.p[1], dz = po.z - sv.p[2];
            j0 -= sv.a[1] * dz - sv.a[2] * dy; j1 -= sv.a[2] * dx - sv.a[0] * dz; j2 -= sv.a[0] * dy - sv.a[1] * dx;
          } else { j0 -= sv.a[0]; j1 -= sv.a[1]; j2 -= sv.a[2]; }
        }
      }
      float gx, gy, gz;
      if (dm.loss == DEXR_LOSS_POSITION) {
        const float ax_ = fabsf(rx), ay_ = fabsf(ry), az_ = fabsf(rz);
        const float wx = ax_ < beta ? inv_beta : fast_rcp(ax_);
        const float wy = ay_ < beta ? inv_beta : fast_rcp(ay_);
        const float wz = az_ < beta ? inv_beta : fast_rcp(az_);
        gx = T.w * rx * wx; gy = T.w * ry * wy; gz = T.w * rz * wz;
      } else {
        const float d = sqrtf(fmaf(rx, rx, fmaf(ry, ry, rz * rz)));
        const float invd = d > 1e-30f ? fast_rcp(d) : 0.f;
        const float hp = d < beta ? d * inv_beta : 1.0f;
        gx = T.w * hp * (rx * invd); gy = T.w * hp * (ry * invd); gz = T.w * hp * (rz * invd);
      }
      g = fmaf(j0, gx, fmaf(j1, gy, fmaf(j2, gz, g)));
    }
    // mimic fold g_x = M^T g_q (kinematics_adaptor.py backward_jacobian), as in solve()
    if (dm.has_mimic) {
      const int gcount = st.group_count[l];
      float gx_ = 0.f;
#pragma unroll
      for (int k = 0; k < DEXR_MAX_GROUP; ++k) {
        const bool v = isvar && k < gcount;
        const float gv = gshfl<G>(g, v ? st.group_lane[l][k] : l);
        if (v) gx_ = fmaf(st.group_mult[l][k], gv, gx_);
      }
      g = gx_;
    }
    g = isvar ? fmaf(2.0f * sv.prm.norm_delta, x - x0, g) : 0.f;
  }
  if (active) {
    if (isvar && io.grad_out) io.grad_out[f * dm.n_var + sv.var] = g;
    if (l == 0) {
      if (io.loss_out) io.loss_out[f] = loss;
      if (io.cost_out) io.cost_out[f] = cost;
    }
  }
  __syncwarp();  // the group's next frame rewrites the targets and link positions this one read
}

}  // namespace dexr
