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
// with cp.async.bulk (TMA 1-D) into a ring of up to four stages guarded by mbarriers; the CTAs claim tiles from a
// grid-wide queue, and consumer warps claim frames from the ring dynamically.
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

// v, passed through an empty asm the compiler cannot look into or move: what is derived from the result is computed where it
// is used instead of being hoisted out of the frame loop as a loop invariant and held in a register through every frame.
// No instruction is emitted.
__device__ __forceinline__ uint32_t opaque(uint32_t v) {
#ifndef DEXR_HOST_EMULATION
  asm volatile("" : "+r"(v));
#endif
  return v;
}
__device__ __forceinline__ long long opaque(long long v) {
#ifndef DEXR_HOST_EMULATION
  asm volatile("" : "+l"(v));
#endif
  return v;
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
#ifndef DEXR_HOST_EMULATION
  __syncwarp();  // lanes 0-15 of warp 0 wrote the link and residual arrays that thread 0 reads below
#endif
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
      // Thread 0 runs this part alone while the CTA waits: it counts and schedules from the shared copies of the link
      // parents, masks and residual links, not through chains of dependent global loads (links on the same lane as link
      // k, for every link k on a lane: parents are < dof <= 32, -1 for the world).
      const int nl = tb->n_links;
      int mx = 0;
      DEXR_ROLL for (int k = 0; k < nl; ++k) {
        const int pk = __float_as_int(st.link_off[k].w);
        int n = 0;
        DEXR_ROLL for (int j = 0; j < nl; ++j) n += (__float_as_int(st.link_off[j].w) == pk);
        if (pk >= 0) mx = n > mx ? n : mx;
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
          const int rt = st.res_task[k], ro = st.res_origin[k];
          const uint32_t msk = st.link_anc[rt] | (ro >= 0 ? st.link_anc[ro] : 0u);
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
// BW: the Solver<G, BW> instantiation the group runs.  Block mode (BW > 0) backs up only the BW-column row segments its
// lanes hold and factorises every block in registers, so it needs no transposed factor: its last area holds the NP
// right-hand sides instead (2.1 KB instead of 3.9 KB per 16-lane group: room for more consumer warps next to the ring);
// dense mode needs all NP rows (and the mimic-fold temporaries), arrow mode keeps its Schur matrix in the backup area.
template <int G, int BW = 0>
struct Scratch {
  static constexpr int NP = G;
  static constexpr int kRows = BW > 0 ? BW : NP;                // rows of the backup
  static constexpr int kFr = 0;                                 // [MAX_RES][4] target xyz, weight c_k
  static constexpr int kLp = kFr + DEXR_MAX_RES * 4;            // [2][MAX_LINKS][4] link positions
  static constexpr int kU = kLp + 2 * DEXR_MAX_LINKS * 4;       // jbuf[2][3][NP] (aliased by the 2 Cholesky row buffers) + at: 2 x [NP + NP/4] float4
  static constexpr int kUSize = 16 * NP;
  static constexpr int kHb = kU + kUSize;                       // [kRows][NP]   Hessian backup, column per lane
  static constexpr int kLcol = kHb + kRows * NP;                // [NP][NP+1] L^T rows, conflict-free column reads (also mimic-fold temp)
  static constexpr int kRhs = kLcol;                            // block mode: [NP] -g of every lane, the blocks' right-hand sides
  static constexpr int kFloats = ((kLcol + (BW > 0 ? NP : kRows * (NP + 1)) + 3) / 4) * 4;
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

// The integer and boolean bookkeeping of Solver::solve (group-uniform).  Packed (the 16-lane block-diagonal solver, whose
// frames kernel runs at 80 registers): two words instead of eleven registers carried through every phase of an iteration.
//   w0: bits 0-15 iterations, 16-22 rejected trials (saturated at 127), 23-25 the status flags, 26 done, 27 exact,
//       28 recheck, 29 trust_prev, 30-31 stall (saturated at 3: only `stall >= 2` is read)
//   w1: bits 0-15 the free-variable mask of the previous iteration, 16-30 rechecks (at most 3), 31 the step accepted in this
//       iteration was below kNearStep (kNear: inc_rechecks() masks it out of the count)
// w0 & 0x3ffffff is the status word (dexr.h).  Unpacked: one variable each.
template <bool P>
struct Bookkeeping {
  static constexpr uint32_t kDone = 1u << 26, kExact = 1u << 27, kRecheck = 1u << 28, kTrust = 1u << 29;
  static constexpr uint32_t kNear = 1u << 31;  // (w1)
  uint32_t w0 = kExact, w1 = 0;
  int iters_ = 0, rejects_ = 0, rechecks_ = 0, stall_ = 0, status_ = 0;
  unsigned last_fmask_ = 0u;
  bool done_ = false, exact_ = true, recheck_ = false, trust_ = false;

  __device__ __forceinline__ bool get(uint32_t bit, bool v) const { return P ? (w0 & bit) != 0u : v; }
  __device__ __forceinline__ void put(uint32_t bit, bool& v, bool x) {
    if constexpr (P) w0 = x ? (w0 | bit) : (w0 & ~bit);
    else v = x;
  }
  __device__ __forceinline__ bool done() const { return get(kDone, done_); }
  __device__ __forceinline__ void set_done(bool x) { put(kDone, done_, x); }
  __device__ __forceinline__ bool exact() const { return get(kExact, exact_); }
  __device__ __forceinline__ void set_exact(bool x) { put(kExact, exact_, x); }
  __device__ __forceinline__ bool recheck() const { return get(kRecheck, recheck_); }
  __device__ __forceinline__ void set_recheck(bool x) { put(kRecheck, recheck_, x); }
  __device__ __forceinline__ bool trust_prev() const { return get(kTrust, trust_); }
  __device__ __forceinline__ void set_trust_prev(bool x) { put(kTrust, trust_, x); }
  __device__ __forceinline__ void flag(int s) {
    if constexpr (P) w0 |= (uint32_t)s;
    else status_ |= s;
  }
  __device__ __forceinline__ int iters() const { return P ? (int)(w0 & 0xffffu) : iters_; }
  __device__ __forceinline__ void inc_iters() {  // (max_iters <= 65535: the field does not wrap)
    if constexpr (P) ++w0;
    else ++iters_;
  }
  __device__ __forceinline__ void inc_rejects() {
    if constexpr (P) { if ((w0 & (0x7fu << 16)) != (0x7fu << 16)) w0 += 1u << 16; }
    else ++rejects_;
  }
  __device__ __forceinline__ int stall() const { return P ? (int)(w0 >> 30) : stall_; }
  __device__ __forceinline__ void clear_stall() {
    if constexpr (P) w0 &= ~(3u << 30);
    else stall_ = 0;
  }
  __device__ __forceinline__ void inc_stall() {
    if constexpr (P) { if ((w0 >> 30) != 3u) w0 += 1u << 30; }
    else ++stall_;
  }
  __device__ __forceinline__ unsigned last_fmask() const { return P ? (w1 & 0xffffu) : last_fmask_; }
  __device__ __forceinline__ void set_last_fmask(unsigned m) {
    if constexpr (P) w1 = (w1 & ~0xffffu) | m;
    else last_fmask_ = m;
  }
  // packed only (the unpacked solver keeps the accepted step itself)
  __device__ __forceinline__ bool near() const { return (w1 & kNear) != 0u; }
  __device__ __forceinline__ void set_near(bool x) { w1 = x ? (w1 | kNear) : (w1 & ~kNear); }
  __device__ __forceinline__ int inc_rechecks() {  // ++rechecks
    if constexpr (P) { w1 += 1u << 16; return (int)((w1 >> 16) & 0x7fffu); }
    else return ++rechecks_;
  }
  // the status word: flags, iterations and rejected trials (saturated at 127)
  __device__ __forceinline__ int status() const {
    if constexpr (P) return (int)(w0 & 0x3ffffffu);
    else return status_ | ((iters_ & 0xffff) | ((rejects_ > 127 ? 127 : rejects_) << 16));
  }
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
  using SC = Scratch<G, BW>;

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
#ifdef DEXR_EXP_TIMELINE
  long long issued = 0;       // outer iterations this group's warp has run, masked ones included (tools/frames_timeline.py)
#else
  static constexpr long long issued = 0;
#endif

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
    if constexpr (BW > 0) {
      static_assert(BW <= 0 || G == 16, "the packed lane constants hold 16-lane masks");
      lane_pk = (uint32_t)lane | ((uint32_t)(var + 1) << 5) | ((jtype != 0 ? 1u : 0u) << 10) | ((sc_off >> 4) << 12);
      mask_pk = (anc & 0xffffu) | (desc << 16);
    }
  }

  // The block-diagonal frames kernel runs 24 warps per SM at 80 registers (dexr.cu, frames_warps()).  There the lane's integer
  // constants (lane index, scratch offset, ancestor / descendant masks, variable index, joint type) are kept packed in two
  // words, lane_pk and mask_pk, which pass through opaque() at the top of every frame, iteration, trial and fallback pass
  // and after the trial FK; the members are unpacked from them there.  So two registers carry the constants from one phase
  // to the next, and the shared-memory addresses, masks and predicates derived from them are recomputed where they are used
  // (a few integer instructions) instead of being held in registers -- or spilled -- from one use to the next.
  //   lane_pk: bits 0-4 lane, 5-9 var + 1, 10 jtype != 0 (only `jtype == 0` is read), 12-31 sc_off / 16
  //   mask_pk: bits 0-15 anc, 16-31 desc
  // Other instantiations are unchanged.
  uint32_t lane_pk = 0u, mask_pk = 0u;
  __device__ __forceinline__ void refresh() {
    if constexpr (BW > 0) {
      lane_pk = opaque(lane_pk); mask_pk = opaque(mask_pk);
      lane = (int)(lane_pk & 31u); l = lane & (G - 1);
      var = (int)((lane_pk >> 5) & 31u) - 1; jtype = (int)((lane_pk >> 10) & 1u);
      sc_off = (lane_pk >> 12) << 4;
      anc = mask_pk & 0xffffu; desc = mask_pk >> 16;
    }
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
  // the transposed factor (dense, arrow) or the mimic-fold temporary (dense); block mode has no such area: there kLcol is kRhs
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
  __device__ __forceinline__ void world_axis(const float* Rw, float* ax) const {
    const float ax0 = ST().lane_c[6][l].w, ax1 = ST().lane_c[7][l].w, ax2 = ST().lane_c[8][l].w;
    ax[0] = fmaf(Rw[0], ax0, fmaf(Rw[1], ax1, Rw[2] * ax2));
    ax[1] = fmaf(Rw[3], ax0, fmaf(Rw[4], ax1, Rw[5] * ax2));
    ax[2] = fmaf(Rw[6], ax0, fmaf(Rw[7], ax1, Rw[8] * ax2));
  }
  __device__ __forceinline__ void set_world_axis(const float* Rw) { world_axis(Rw, a); }

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
    Bookkeeping<(BW > 0 && G == 16)> bk;
    refresh();

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
      bk.flag(DEXR_STATUS_NONFINITE);
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
    bk.set_done(!active);
    // Curvature model (group-uniform): `exact` = use the true second derivative of the norm-Huber loss
    // (radial direction has zero curvature beyond beta); otherwise its quadratic majoriser 1/d * I, which
    // is positive semi-definite and globally safer.  Optimistic start, demoted after a large or failed step.
    // A tiny accepted step ends the frame -- unless some variable is held at a bound: then the gradient is
    // re-evaluated once more, and the frame ends only if the same set stays active (KKT on the bounds).
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

    while (gany<32>(!bk.done(), lane)) {
#ifdef DEXR_EXP_TIMELINE
      ++issued;
#endif
      refresh();
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
          const float s_rad = (quad || !bk.exact()) ? 0.f : T.w * invd;
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
      if (bk.recheck() && (fmask == bk.last_fmask() || bk.inc_rechecks() >= 3)) bk.set_done(true);
      bk.set_recheck(false);
      bk.set_last_fmask(fmask);
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
      if (bk.trust_prev() && !bk.done()) {
        if (gn < gn_prev) {
          if (gn < kTrustDecrease * gn_prev) lam = fmaxf(lam * kLamDown, kLamMin);
          bk.clear_stall();
        } else {
          revert = true;
          bk.inc_stall();
        }
      }
      DEXR_TRACE_PRINT("  it %2d gn %.3e gn_prev %.3e trust_prev %d stall %d revert %d lam %.1e\n", bk.iters(), gn, gn_prev, (int)bk.trust_prev(), bk.stall(), (int)revert, lam);
      float* hbuf = hb();
#pragma unroll
      for (int i = 0; i < HN; ++i) hbuf[i * NP + l] = H[i];
      if constexpr (BW > 0) scf()[SC::kRhs + l] = -g;  // every lane of a window solves the window's whole block
      // own diagonal entry (register index = lane id is not addressable: read it back from the column store);
      // the regulariser 2*norm_delta enters on the diagonal at pivot time together with the damping
      const float reg2 = free_ ? 2.0f * nd : 0.f;
      const int dj = AR ? (ar_trunk ? 8 + l : l - ar_fb) : l - cb;  // register holding this lane's diagonal entry
      float hd = free_ ? hbuf[dj * NP + l] + reg2 : 1.0f;
      float D = fabsf(hd) + 1e-6f;
      // ======================= damped Newton trials ====================================
      bool accepted = bk.done();
      float acc_step = 0.f;
      float Rn[9], pn[3], an[3];
      for (int trial = 0; trial < kMaxTrials; ++trial) {
        if (!gany<32>(!accepted, lane)) break;
        refresh();
        // (block mode factorises straight from the backup and does not hold H in registers through the trials at all)
        if (BW <= 0 && trial > 0) {
#pragma unroll
          for (int i = 0; i < HN; ++i) H[i] = hbuf[i * NP + l];
        }
        float y = -g;
        float myinv = 1.0f;
        bool bad = false;
        // dense and arrow modes only: two NP-float row buffers, alternating per pivot, and the transposed factor.  Block mode
        // uses neither -- its kLcol area is kRhs, the right-hand sides the block factorisation reads -- and must not write
        // through them.
        float* Lr = lrow();
        float* Lc = lcol();
        __syncwarp();  // (block mode: the backup and right-hand-side stores of the other rows of the window)
        if constexpr (BW > 0) {
          // ================= block factorisation: every window's 4 x 4 block in registers =================
          // Every lane of a window factorises and solves the window's block redundantly (Cholesky, forward and back
          // substitution) from the backup, which holds entry (r, c) of the block as row r stored it -- H is not bitwise
          // symmetric, so only the lower triangle, r >= c, is read, as the dense pivot loop below reads it.  The operations
          // and their order are the pivot loop's for bw = 4, so the step is the same to the bit; what goes away is its
          // per-pivot traffic: two shuffles, two row-buffer stores, a warp barrier and a row load per pivot, and four
          // shuffles and loads in the back substitution.
          static_assert(BW == 4, "the register factorisation is written for 4-joint windows");
          // Written column by column (left looking), the substitutions after the factorisation: every entry sees the same
          // updates in the same order (pivot 0, 1, ...) as in the pivot loop.
          // (the window's first lane is formed from the lane index refresh() just unpacked, not from the iteration's cb: what
          // derives from it -- the rows' free bits and regularisers -- is then formed here rather than held through the trials)
          const int wb = l & ~(BW - 1);
          const float* hw = hb() + wb;  // hw[j * NP + r]: entry (r, j) of this window's block
          // the damping + regulariser row r adds to its pivot, d_r = a_rr + fmaf(lam, D, reg2) with hd, D and reg2 as lane wb + r
          // forms them from its stored diagonal entry hrr
          auto pivot = [&](int r, float hrr, float arr) {
            const bool fr = (fmask >> (wb + r)) & 1u;
            const float rg = fr ? 2.0f * nd : 0.f;
            const float d = arr + fmaf(lam, fabsf(fr ? hrr + rg : 1.0f) + 1e-6f, rg);
            bad = bad || !(d > 1e-20f);
            return fast_rsqrt(fmaxf(d, 1e-20f));
          };
          const float4 c0 = *reinterpret_cast<const float4*>(hw);
          const float i0 = pivot(0, c0.x, c0.x);
          const float l10 = c0.y * i0, l20 = c0.z * i0, l30 = c0.w * i0;
          const float4 c1 = *reinterpret_cast<const float4*>(hw + NP);
          const float i1 = pivot(1, c1.y, fmaf(-l10, l10, c1.y));
          const float l21 = fmaf(-l20, l10, c1.z) * i1, l31 = fmaf(-l30, l10, c1.w) * i1;
          const float4 c2 = *reinterpret_cast<const float4*>(hw + 2 * NP);
          const float i2 = pivot(2, c2.z, fmaf(-l21, l21, fmaf(-l20, l20, c2.z)));
          const float l32 = fmaf(-l31, l21, fmaf(-l30, l20, c2.w)) * i2;
          const float h33 = hw[3 * NP + 3];
          const float i3 = pivot(3, h33, fmaf(-l32, l32, fmaf(-l31, l31, fmaf(-l30, l30, h33))));
          // forward substitution, L z = -g
          const float4 rhs = *reinterpret_cast<const float4*>(scf() + SC::kRhs + wb);
          const float z0 = rhs.x * i0;
          const float z1 = fmaf(-l10, z0, rhs.y) * i1;
          const float z2 = fmaf(-l21, z1, fmaf(-l20, z0, rhs.z)) * i2;
          const float z3 = fmaf(-l32, z2, fmaf(-l31, z1, fmaf(-l30, z0, rhs.w))) * i3;
          // back substitution, L^T delta = z
          const float x3 = z3 * i3;
          const float x2 = fmaf(-l32, x3, z2) * i2;
          const float x1 = fmaf(-l21, x2, fmaf(-l31, x3, z1)) * i1;
          const float x0 = fmaf(-l10, x1, fmaf(-l20, x2, fmaf(-l30, x3, z0))) * i0;
          const int r = l - wb;
          y = r == 0 ? x0 : (r == 1 ? x1 : (r == 2 ? x2 : x3));
        }
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
        if constexpr (dense) {
          // One pivot step, with the number of 4-column chunks of the rotating window it updates fixed at compile time.  The
          // window shrinks by one column per pivot, so the steps are run in PHASES of decreasing chunk count (HN = 16: 4, 3,
          // 2, 1 chunks while more than 12, 8, 4, 0 columns are live) instead of predicating all HN / 4 chunks off one by
          // one: half of the FFMA / LDS.128 issue slots of a 16 x 16 factorisation went into predicated-off instructions.
          constexpr int kMask = NP - 1;
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
          } else {
            static_assert(HN == 16 || HN == 32, "dense groups are 16 or 32 lanes");
          }
        }
        // back substitution: L^T delta = y (column oriented, transposed copy read conflict free)
        for (int k = (dense ? bw : 0) - 1; k >= 0; --k) {
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
            refresh();
            const float4 a_self = at_a(l);          // (rev ? a : 0), t of this lane, as stored when H was built
            const float4 t_self = at_t(l);
#pragma unroll
            for (int j = 0; j < HN; ++j) {
              if (AR ? (j < 8 ? j < ar_maxw : j - 8 < ar_t) : j < bw) {
                const int i = AR ? (j < 8 ? (ar_fb + j < NP ? ar_fb + j : NP - 1) : j - 8) : (BW > 0 ? (l & ~(BW - 1)) : cb) + j;
                const float4 ai = at_a(i);
                const float4 ti_ = at_t(i);
                const bool up = (anc >> i) & 1u;
                const bool dn = (desc >> i) & 1u;
                const float vu = fmaf(ai.x, t_self.x, fmaf(ai.y, t_self.y, ai.z * t_self.z));
                const float vd = fmaf(a_self.x, ti_.x, fmaf(a_self.y, ti_.y, a_self.z * ti_.z));
                const bool mine = !AR || (j < 8 ? j < ar_fw : true);
                const float v = mine ? (up ? vu : (dn ? vd : 0.f)) : 0.f;
                // same column bookkeeping as the freeze pass: frozen rows / columns stay zero (identity)
                // (block mode: the window base from the lane index refresh() unpacked, as in the factorisation)
                const int cj = AR ? (j < 8 ? (j < ar_fw ? ar_fb + j : -1) : (j - 8 < ar_t ? j - 8 : -1)) : (BW > 0 ? (l & ~(BW - 1)) : cb) + j;
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
          if (!accepted && !dropped) { lam *= kLamUp; bk.inc_rejects(); }
          continue;
        }
        float xn = free_ ? fminf(fmaxf(x + y, lo), hi) : x;
        if (bad) xn = x;
        if (revert) xn = x_prev;  // (every lane: the variable set that was free during the reverted step may differ)
        const float dx = xn - x;
        // the step's length and the quadratic model's predicted decrease (block mode: after the trial point's FK and cost, so
        // that they are not held through them; D of this lane's row is formed again from the backup, as the factorisation
        // forms its rows' shifts, instead of being held through the trials)
        float step, pred;
        if constexpr (BW <= 0) {
          step = gmax<G>(fabsf(dx));
          pred = 0.5f * gsum<G>(dx * fmaf(lam * D, dx, -g));
        }
        const float qn = compose_q(xn);
        fk(qn, Rn, pn);
        refresh();
        write_links(Rn, pn, cur ^ 1);
        // block mode: the trial point's world axis right away, so that its 3x3 rotation is dead through cost() and the
        // acceptance test (6 live registers fewer; the same operations, also on a rejected trial)
        if constexpr (BW > 0) world_axis(Rn, an);
        __syncwarp();
        cost(cur ^ 1, xn);
        if constexpr (BW > 0) {
          step = gmax<G>(fabsf(dx));
          const float Dl = fabsf(free_ ? hb()[(l & (BW - 1)) * NP + l] + reg2 : 1.0f) + 1e-6f;
          pred = 0.5f * gsum<G>(dx * fmaf(lam * Dl, dx, -g));
        }
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
        DEXR_TRACE_PRINT("  it %2d trial %d lam %.1e exact %d step %.3e pred %.3e F %.9e Fn %.9e dF %.2e noise %.1e bad %d ok %d ver %d fmask %x\n", bk.iters(),
                         trial, lam, (int)bk.exact(), step, pred, F, Fn, dF, fnoise, (int)bad, (int)ok, (int)verified, fmask);
        if (!accepted) {
          if (ok) {
            x_prev = x;
            x = xn; q = qn; F = Fn;
            Fnz = cost_nz;
            Fl = cost_lane;
            if constexpr (BW > 0) {
#pragma unroll
              for (int i = 0; i < 3; ++i) a[i] = an[i];
            } else {
              set_world_axis(Rn);
            }
#pragma unroll
            for (int i = 0; i < 3; ++i) p[i] = pn[i];
            cur ^= 1;
            // (see kStopAhead; not with active bounds, extra damping or the majoriser model in play)
            const bool ahead = bk.exact() && !any_act && trial == 0 && !revert && lam <= prm.lambda0 &&
                               step * fmaxf(step, kStopAheadRate * s_prev) < kStopAhead * prm.tol * s_prev;
            s_prev = (trial == 0 && !revert) ? step : 0.f;
            if (bk.iters() == 0 && !revert) lam_carry = fmaxf(prm.lambda0, kCarry * lam);
            if (verified) lam = fmaxf(lam * kLamDown, kLamMin);
            if (verified && fabsf(dF + pred) <= kModelGood * pred) lam = fmaxf(lam * kLamDown, kLamMin);  // (kModelGood)
            // fnoise is a worst-case bound (every rounding error with the same sign); a decrease beyond an eighth of it is
            // already unlikely to be noise: such a step is kept whatever the next gradient says (it just does not relax
            // the damping).  Only steps whose effect on F is truly unresolved are put to the gradient test.
            bk.set_trust_prev(!verified && !revert && !(dF < -0.125f * fnoise));
            if (verified) bk.clear_stall();
            gn_prev = gn;
            accepted = true;
            if constexpr (BW > 0) bk.set_near(step < kNearStep);  // (a bit of the packed bookkeeping instead of a register)
            else acc_step = step;
            if (revert) {  // back at the previous point: more damping, or the end when this is the second revert in a row
              lam *= kLamUp;
              bk.inc_rejects();
              if (bk.stall() >= 2) { bk.set_done(true); bk.flag(DEXR_STATUS_NOISEFLOOR); }
              revert = false;
            } else if (step < prm.tol || ahead) {
              if (any_act) bk.set_recheck(true);
              else bk.set_done(true);
            }
          } else {
            if (!dropped)
            {
              lam *= kLamUp;
              bk.inc_rejects();
            }
          }
        }
        __syncwarp();
      }
      if (!bk.done()) {
        if (!accepted) {
          if (bk.exact()) lam = prm.lambda0;  // retry this point with the majoriser model
          else bk.set_done(true);             // no descent direction left at fp32 resolution
        }
        bk.set_exact(accepted && (BW > 0 ? bk.near() : acc_step < kNearStep));
        bk.inc_iters();
        if (bk.iters() >= prm.max_iters && !bk.done()) { bk.set_done(true); bk.flag(DEXR_STATUS_MAXITER); }
      }
    }
    return bk.status();
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
  if constexpr (BW > 0) f = opaque(f);  // (the output addresses are formed here, not held through the solve: see Solver::refresh)
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
// REC (dexr_solve_sequences_tape): the writing group also stores every frame's unfiltered solution to `tape_qpos` and, for
// DexPilot, the flags the frame left to `tape_proj` -- two extra stores on the same code path, so the results do not change.
template <int G, int BW, bool REC = false>
__device__ __forceinline__ void solve_stream(Solver<G, BW>& sv, const dexr_sequences_t& io, const Dims& dm,
                                             const dexr_params_t& prm, const long long& S, const int& steps, long long s,
                                             bool active, bool writes, float* kpbuf, bool use_filter,
                                             float* tape_qpos = nullptr, uint8_t* tape_proj = nullptr) {
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
    if constexpr (REC) {
      if (writes) {  // (lane l < len_proj wrote flag l of the stream's buffer in prepare_targets)
        const long long fr = sc * steps + t;
        if (sv.var >= 0) tape_qpos[fr * dm.n_var + sv.var] = last;
        if (tape_proj && l < dm.len_proj) tape_proj[fr * dm.len_proj + l] = io.projected[sc * dm.len_proj + l];
      }
    }
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

// ------------------------------------------------------------------------------------------------
// backpropagation through the solve (dexr_solve_vjp): implicit-function cotangents at a given point
// ------------------------------------------------------------------------------------------------
// At a stationary point x of F(x; theta) = L(x; theta) + norm_delta |x - a|^2 on its free variables, g(x*(theta); theta) = 0
// gives dx*/dtheta = -H_ff^-1 dg_f/dtheta, so for a cotangent gbar = dl/dx: v_f = H_ff^-1 gbar_f, v_A = 0 on the active
// variables, and theta_bar = -(dg/dtheta)^T v.  H is the EXACT Hessian of F -- not the solver's curvature models (no position
// majoriser, no dropped radial term, no positive-definite fallback, no damping) -- so this runs on its own Hessian code
// rather than solve()'s; sharing code with solve() would also change the solver kernels' machine code.  The Jacobian-column
// and loss-derivative formulas are those of evaluate_frame, restated in vjp_column rather than factored out of it, so that the
// evaluation kernels' machine code stays untouched.
//
// Per-group scratch (floats), the dense Scratch<G> layout up to kLcol followed by three small arrays:
//   kFr, kLp   targets and link positions, as in a solve (one link buffer used)
//   kU         jbuf[2][3][NP]: the lanes' Jacobian columns of the residual in flight; at_a / at_t: axis and torque sums of
//              the kinematic curvature
//   kH         [NP][NP] H_q, the joint-space Hessian of L (loss + kinematic curvature), column per lane (symmetric)
//   kA         [NP][NP+1] M^T H_q M + 2 norm_delta I over the free variables, identity rows and columns elsewhere; row per
//              lane, factorised in place (lower Cholesky factor)
//   kMv        [NP] M v: the solution mapped to joint space (mimic lanes get mult * v of their source, fixed lanes 0)
//   kKp        [64] the keypoint cotangent accumulator
//   kFlags     16 bytes: the frame's DexPilot flags.  prepare_targets writes back the flags it reads; it gets this private
//              copy, so the caller's `projected` is never written
// 16 lanes: 1060 floats (4.1 KB) per group; 32 lanes: 2884 floats (11.3 KB).
template <int G>
struct VjpScratch {
  static constexpr int NP = G;
  static constexpr int kH = Scratch<G>::kHb;
  static constexpr int kA = Scratch<G>::kLcol;
  static constexpr int kMv = kA + NP * (NP + 1);
  static constexpr int kKp = kMv + NP;
  static constexpr int kFlags = kKp + 64;
  static constexpr int kFloats = ((kFlags + 4 + 3) / 4) * 4;
};
static_assert(VjpScratch<16>::kFloats == 1060 && VjpScratch<32>::kFloats == 2884, "VJP scratch layout (DESIGN.md 3.8)");

// The argument checks of dexr_solve_vjp that read the robot's table: nullptr, or what is wrong.  Host code shared by the
// library and the host emulation, as eval_io_error.
inline const char* vjp_io_error(const dexr_table_t& t, const dexr_vjp_t& io, const dexr_params_t& prm) {
  if (!io.qpos) return "qpos is required";
  if (!io.grad_qpos) return "grad_qpos is required";
  if ((io.keypoints != nullptr) == (io.ref_value != nullptr)) return "exactly one of keypoints / ref_value must be given";
  if (prm.preprocess != 0) return "raw-landmark pre-processing is not differentiated: params.preprocess must be 0";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  if (io.grad_keypoints && !io.keypoints) return "grad_keypoints needs the keypoints form";
  if (io.grad_ref_value && !io.ref_value) return "grad_ref_value needs the ref_value form";
  if (io.grad_last_qpos && !io.last_qpos) return "grad_last_qpos needs last_qpos";
  return nullptr;
}

// This lane's Jacobian column of residual k (task minus origin link) and the residual r = p_task - p_origin - target.
template <int G>
__device__ __forceinline__ void vjp_column(const Solver<G, 0>& sv, int k, float& j0, float& j1, float& j2, float& rx,
                                           float& ry, float& rz) {
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l;
  const bool rev = sv.jtype == 0;
  const int ti = st.res_task[k], oi = st.res_origin[k];
  const float4 T = sv.fr()[k];
  const float4 pt = sv.lp(0)[ti];
  rx = pt.x - T.x; ry = pt.y - T.y; rz = pt.z - T.z;
  j0 = 0.f; j1 = 0.f; j2 = 0.f;
  if ((st.link_anc[ti] >> l) & 1u) {
    if (rev) {
      const float dx = pt.x - sv.p[0], dy = pt.y - sv.p[1], dz = pt.z - sv.p[2];
      j0 = sv.a[1] * dz - sv.a[2] * dy; j1 = sv.a[2] * dx - sv.a[0] * dz; j2 = sv.a[0] * dy - sv.a[1] * dx;
    } else { j0 = sv.a[0]; j1 = sv.a[1]; j2 = sv.a[2]; }
  }
  if (oi >= 0) {
    const float4 po = sv.lp(0)[oi];
    rx -= po.x; ry -= po.y; rz -= po.z;
    if ((st.link_anc[oi] >> l) & 1u) {
      if (rev) {
        const float dx = po.x - sv.p[0], dy = po.y - sv.p[1], dz = po.z - sv.p[2];
        j0 -= sv.a[1] * dz - sv.a[2] * dy; j1 -= sv.a[2] * dx - sv.a[0] * dz; j2 -= sv.a[0] * dy - sv.a[1] * dx;
      } else { j0 -= sv.a[0]; j1 -= sv.a[1]; j2 -= sv.a[2]; }
    }
  }
}

// The data part of the exact Hessian and gradient at the point the group's scratch holds (targets in kFr, links of the FK at
// x in lp(0), this lane's world axis and origin in sv.a / sv.p): H_q (loss curvature J^T (d2h/dr2) J plus the kinematic
// curvature, column per lane) is written to the scratch's kH, and M^T g_q -- the gradient of L folded onto the variables
// (meaningful on variable lanes only) -- is returned.  Shared by vjp_front and the smoother's forward sweep.  `kin` false leaves
// the kinematic curvature out of H_q: the Gauss-Newton model J^T (d2h/dr2) J, positive semi-definite (the smoother's fallback
// when the exact model is indefinite); the gradient is the same.
template <int G>
__device__ __forceinline__ float exact_grad_hq(Solver<G, 0>& sv, const Dims& dm, bool kin = true) {
  using VS = VjpScratch<G>;
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, dof = dm.dof, m = dm.n_res;
  const bool isvar = sv.var >= 0;
  float* const hq = sv.scf() + VS::kH;

  // ---- gradient of L and H_q, one residual per pass: loss curvature J^T (d2h/dr2) J, then the kinematic curvature
  const float beta = sv.prm.huber_delta, inv_beta = sv.inv_beta;
  const bool pos_loss = dm.loss == DEXR_LOSS_POSITION;
  float H[NP];
#pragma unroll
  for (int i = 0; i < NP; ++i) H[i] = 0.f;
  float g = 0.f, t0 = 0.f, t1 = 0.f, t2 = 0.f;
  for (int k = 0; k < m; ++k) {
    float j0, j1, j2, rx, ry, rz;
    vjp_column(sv, k, j0, j1, j2, rx, ry, rz);
    const float w = sv.fr()[k].w;
    float gx, gy, gz, y0, y1, y2;  // dh/dr and (d2h/dr2) j
    if (pos_loss) {
      // per-coordinate Huber: curvature w / beta inside the quadratic zone, exactly 0 beyond it
      const float ax_ = fabsf(rx), ay_ = fabsf(ry), az_ = fabsf(rz);
      gx = w * rx * (ax_ < beta ? inv_beta : fast_rcp(ax_));
      gy = w * ry * (ay_ < beta ? inv_beta : fast_rcp(ay_));
      gz = w * rz * (az_ < beta ? inv_beta : fast_rcp(az_));
      y0 = ax_ < beta ? w * inv_beta * j0 : 0.f;
      y1 = ay_ < beta ? w * inv_beta * j1 : 0.f;
      y2 = az_ < beta ? w * inv_beta * j2 : 0.f;
    } else {
      // Huber of the norm: w I / beta for d < beta, w (I - u u^T) / d beyond (the radial curvature is exactly 0 there)
      const float d = sqrtf(fmaf(rx, rx, fmaf(ry, ry, rz * rz)));
      const bool quad = d < beta;
      const float invd = d > 1e-30f ? fast_rcp(d) : 0.f;
      const float ux = rx * invd, uy = ry * invd, uz = rz * invd;
      const float hp = quad ? d * inv_beta : 1.0f;
      gx = w * hp * ux; gy = w * hp * uy; gz = w * hp * uz;
      const float s_iso = w * (quad ? inv_beta : invd);
      const float uj = (quad ? 0.f : w * invd) * fmaf(ux, j0, fmaf(uy, j1, uz * j2));
      y0 = fmaf(s_iso, j0, -uj * ux); y1 = fmaf(s_iso, j1, -uj * uy); y2 = fmaf(s_iso, j2, -uj * uz);
    }
    g = fmaf(j0, gx, fmaf(j1, gy, fmaf(j2, gz, g)));
    t0 += j1 * gz - j2 * gy; t1 += j2 * gx - j0 * gz; t2 += j0 * gy - j1 * gx;
    const int b = k & 1;
    sv.jbuf(b, 0)[l] = j0; sv.jbuf(b, 1)[l] = j1; sv.jbuf(b, 2)[l] = j2;
    __syncwarp();
#pragma unroll
    for (int c4 = 0; c4 < NP; c4 += 4) {
      const float4 c0 = *reinterpret_cast<const float4*>(sv.jbuf(b, 0) + c4);
      const float4 c1 = *reinterpret_cast<const float4*>(sv.jbuf(b, 1) + c4);
      const float4 c2 = *reinterpret_cast<const float4*>(sv.jbuf(b, 2) + c4);
      H[c4 + 0] = fmaf(c0.x, y0, fmaf(c1.x, y1, fmaf(c2.x, y2, H[c4 + 0])));
      H[c4 + 1] = fmaf(c0.y, y0, fmaf(c1.y, y1, fmaf(c2.y, y2, H[c4 + 1])));
      H[c4 + 2] = fmaf(c0.z, y0, fmaf(c1.z, y1, fmaf(c2.z, y2, H[c4 + 2])));
      H[c4 + 3] = fmaf(c0.w, y0, fmaf(c1.w, y1, fmaf(c2.w, y2, H[c4 + 3])));
    }
  }
  {
    // kinematic curvature (as in solve()): S[l][i] = a_i . t_l for i ancestor-or-self of l, a_l . t_i for i below l, with
    // t_c = sum_k J_kc x dh/dr_k and a the world axis of a revolute joint (0 for a prismatic one)
    const bool rev = sv.jtype == 0;
    const float ar0 = rev ? sv.a[0] : 0.f, ar1 = rev ? sv.a[1] : 0.f, ar2 = rev ? sv.a[2] : 0.f;
    sv.at_a(l) = make_float4(ar0, ar1, ar2, 0.f);
    sv.at_t(l) = make_float4(t0, t1, t2, 0.f);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      if (i < dof) {
        const float4 ai = sv.at_a(i), ti_ = sv.at_t(i);
        const bool up = (sv.anc >> i) & 1u, dn = (sv.desc >> i) & 1u;
        const float vu = fmaf(ai.x, t0, fmaf(ai.y, t1, ai.z * t2));
        const float vd = fmaf(ar0, ti_.x, fmaf(ar1, ti_.y, ar2 * ti_.z));
        H[i] += kin ? (up ? vu : (dn ? vd : 0.f)) : 0.f;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NP; ++i) hq[i * NP + l] = H[i];
  // g_x = M^T g_q, as in evaluate_frame
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
  return g;
}

// Row l of A = the free block of M^T H_q M + diag I (H_q in the scratch's kH, M the scatter + mimic map: lane c's variable
// feeds the joints st.group_lane[c][.] with multipliers st.group_mult[c][.]), identity rows and columns where a variable is
// not free (`fmask`, group-wide) or a lane is not a variable.  Shared by vjp_front (diag = 2 norm_delta) and the smoother.
template <int G>
__device__ __forceinline__ void fold_free_block(const Solver<G, 0>& sv, const Dims& dm, float* A, bool free_, unsigned fmask,
                                                float diag) {
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, dof = dm.dof;
  const float* const hq = sv.scf() + VjpScratch<G>::kH;
  const int gca = free_ ? st.group_count[l] : 0;
  for (int c = 0; c < dof; ++c) {
    float h = c == l ? 1.0f : 0.f;
    if (free_ && ((fmask >> c) & 1u)) {
      h = c == l ? diag : 0.f;
      const int gcb = st.group_count[c];
      for (int fb = 0; fb < gcb; ++fb) {
        const float* col = hq + st.group_lane[c][fb] * NP;
        const float mb = st.group_mult[c][fb];
        for (int fa = 0; fa < gca; ++fa) h = fmaf(mb * st.group_mult[l][fa], col[st.group_lane[l][fa]], h);
      }
    }
    A[l * (NP + 1) + c] = h;
  }
}

// In-place Cholesky of the [dof][NP+1] row-per-lane matrix A (lane = row, one pivot column per step, fp32, IEEE sqrt and
// division): the lower factor.  Returns whether a pivot was <= 0 (group-uniform).  Shared by vjp_front and the smoother.
template <int G>
__device__ __forceinline__ bool factor_rows(float* A, int dof, int l) {
  constexpr int NP = G;
  bool bad = false;
  for (int k = 0; k < dof; ++k) {
    __syncwarp();
    const float d = A[k * (NP + 1) + k];
    bad = bad || !(d > 0.f);  // a pivot <= 0: not a strict local minimum of the free subproblem
    const float lkk = sqrtf(fmaxf(d, 1e-30f));
    __syncwarp();
    if (l == k) A[k * (NP + 1) + k] = lkk;
    else if (l > k && l < dof) A[l * (NP + 1) + k] /= lkk;
    __syncwarp();
    if (l > k && l < dof) {
      const float lik = A[l * (NP + 1) + k];
      for (int j = k + 1; j <= l; ++j) A[l * (NP + 1) + j] = fmaf(-lik, A[j * (NP + 1) + k], A[l * (NP + 1) + j]);
    }
  }
  return bad;
}

// What vjp_tail hands back to its driver, per lane: v (H_ff^-1 gbar_f on this lane's variable, 0 elsewhere), the fixed-joint
// term H_q[c, :] . M v of a fixed lane (its cotangent is -qbar), and the frame's finite / not-positive-definite verdicts
// (group-uniform).  The keypoint cotangents are in the scratch's kKp accumulator.
struct VjpLane {
  float v, qbar;
  bool finite, bad;
};

// What vjp_front leaves for vjp_tail besides the scratch (H_q in kH, the factor in kA, the flags in kFlags): whether this
// lane's variable is free, and the frame's finite / not-positive-definite verdicts (group-uniform).
struct VjpFront {
  bool free_, finite, bad;
};

// The implicit-function VJP of one frame is vjp_front once, then vjp_tail once per cotangent: vjp_frame (dexr_solve_vjp) and
// vjp_stream (dexr_solve_sequences_vjp) run one tail, jacobian_frame (dexr_solve_jacobian) one per free variable.
//
// The per-frame front: the point x, the anchor x0 of this lane's variable come from the driver, with norm_delta `nd`
// (0: no regulariser) and the frame's DexPilot flags `proj` (read into the scratch; nullptr = all 0); `gbar` only takes
// part in the finiteness verdict.  Prepares the targets on the private flag copy, runs FK, builds the gradient, the active
// set and the exact H_q, folds the mimic joints, freezes the active rows and factorises the free block in place in kA.  The
// caller's flags are never written.
template <int G>
__device__ __forceinline__ VjpFront vjp_front(Solver<G, 0>& sv, const FrameInputs& in_, const Dims& dm, float x, float x0,
                                              float gbar, float nd, const uint8_t* proj, bool active) {
  using VS = VjpScratch<G>;
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, lane = sv.lane, dof = dm.dof;
  const bool isvar = sv.var >= 0;
  float* const A = sv.scf() + VS::kA;
  uint8_t* const flags = reinterpret_cast<uint8_t*>(sv.scf() + VS::kFlags);

  // ---- targets (flags on the private copy), FK at x
  const int fixedi = st.fixed_index[l];
  sv.qfix = (active && fixedi >= 0) ? in_.fixed[fixedi] : 0.f;
  sv.x = x;
  if (l < dm.len_proj) flags[l] = (active && proj) ? proj[l] : (uint8_t)0;
  __syncwarp();
  FrameInputs in = in_;
  in.projected = dm.len_proj > 0 ? flags : nullptr;
  bool finite = isfinite(x) && isfinite(x0) && isfinite(sv.qfix) && isfinite(gbar);
  const bool ok_targets = sv.prepare_targets(in, active);
  finite = !gany<G>(!finite, lane) && ok_targets;
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

  float g = exact_grad_hq(sv, dm);
  g = isvar ? fmaf(2.0f * nd, x - x0, g) : 0.f;

  // ---- active set (the solver's rule at its widened bounds), then A = the free block of M^T H_q M + 2 norm_delta I
  const bool act = isvar && ((x <= sv.lo && g > -kGradNoise) || (x >= sv.hi && g < kGradNoise));
  const bool free_ = isvar && !act;
  const unsigned fmask = gballot<G>(free_, lane);
  __syncwarp();
  fold_free_block(sv, dm, A, free_, fmask, 2.0f * nd);
  // ---- Cholesky of A in place
  const bool bad = factor_rows<G>(A, dof, l);
  __syncwarp();
  return VjpFront{free_, finite, bad};
}

// The per-cotangent tail, after vjp_front on the same frame (`fr` its result, `in_` the frame inputs it was given):
// gbar = dl/dx of this lane's variable.  Solves H_ff v = gbar_f with the factor in kA, maps v to joint space (M v), runs the
// target pass -- the ref_value cotangents go to `grad_ref` ([m,3] of the frame, or nullptr), the keypoint ones to the kKp
// accumulator, which it clears first -- and forms the fixed-joint term; everything but grad_ref goes back to the driver.
// Reads the scratch the front left and writes only kMv and kKp, so it can run any number of times after one front.
// SOLVE false skips the substitution: gbar is v itself (the smoother's VJP solves the stacked system of the whole clip and
// runs only the target pass here, after H_q, the targets and the links of the frame are in the scratch; kA is not read).
template <int G, bool SOLVE = true>
__device__ __forceinline__ VjpLane vjp_tail(Solver<G, 0>& sv, const FrameInputs& in_, const Dims& dm, const VjpFront& fr,
                                            float gbar, float* grad_ref, bool active) {
  using VS = VjpScratch<G>;
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, dof = dm.dof, m = dm.n_res;
  const bool isvar = sv.var >= 0;
  const bool free_ = fr.free_, finite = fr.finite, bad = fr.bad;
  const float* const hq = sv.scf() + VS::kH;
  const float* const A = sv.scf() + VS::kA;
  float* const mvs = sv.scf() + VS::kMv;
  float* const kpacc = sv.scf() + VS::kKp;
  const uint8_t* const flags = reinterpret_cast<const uint8_t*>(sv.scf() + VS::kFlags);
  const FrameInputs& in = in_;
  const int fixedi = st.fixed_index[l];
  const float beta = sv.prm.huber_delta, inv_beta = sv.inv_beta;
  const bool pos_loss = dm.loss == DEXR_LOSS_POSITION;
  for (int e = l; e < 64; e += G) kpacc[e] = 0.f;  // (the driver reads its entries of the previous tail on the same lane)

  // v = A^-1 gbar (forward, then back substitution; frozen rows are identity rows with a zero right-hand side)
  float y = free_ ? gbar : 0.f;
  if constexpr (SOLVE) {
    for (int k = 0; k < dof; ++k) {
      const float yk = gshfl<G>(y, k) / A[k * (NP + 1) + k];
      if (l == k) y = yk;
      else if (l > k && l < dof) y = fmaf(-A[l * (NP + 1) + k], yk, y);
    }
    for (int k = dof - 1; k >= 0; --k) {
      const float vk = gshfl<G>(y, k) / A[k * (NP + 1) + k];
      if (l == k) y = vk;
      else if (l < k) y = fmaf(-A[k * (NP + 1) + l], vk, y);
    }
  }
  const float v = bad ? 0.f : y;
  {
    const float vsrc = gshfl<G>(v, sv.msrc >= 0 ? sv.msrc : l);
    mvs[l] = isvar ? v : (sv.msrc >= 0 ? sv.mmult * vsrc : 0.f);
  }
  __syncwarp();
  const float mv = mvs[l];
  // outputs: NaN for a frame with a non-finite input, 0 for one whose free Hessian is not positive definite
  auto out = [&](float val) { return !finite ? __int_as_float(0x7fc00000) : (bad ? 0.f : val); };

  // ---- targets: t_bar_k = (d2h/dr2)(r_k) J_k M v, then through the target map back to ref_value / keypoints
  const bool by_kp = in.kp != nullptr;
  for (int k = 0; k < m; ++k) {
    float j0, j1, j2, rx, ry, rz;
    vjp_column(sv, k, j0, j1, j2, rx, ry, rz);
    const float u0 = gsum<G>(j0 * mv), u1 = gsum<G>(j1 * mv), u2 = gsum<G>(j2 * mv);  // J_k M v
    const float w = sv.fr()[k].w;
    float b0, b1, b2;
    if (pos_loss) {
      b0 = fabsf(rx) < beta ? w * inv_beta * u0 : 0.f;
      b1 = fabsf(ry) < beta ? w * inv_beta * u1 : 0.f;
      b2 = fabsf(rz) < beta ? w * inv_beta * u2 : 0.f;
    } else {
      const float d = sqrtf(fmaf(rx, rx, fmaf(ry, ry, rz * rz)));
      const bool quad = d < beta;
      const float invd = d > 1e-30f ? fast_rcp(d) : 0.f;
      const float ux = rx * invd, uy = ry * invd, uz = rz * invd;
      const float s_iso = w * (quad ? inv_beta : invd);
      const float uu = (quad ? 0.f : w * invd) * fmaf(ux, u0, fmaf(uy, u1, uz * u2));
      b0 = fmaf(s_iso, u0, -uu * ux); b1 = fmaf(s_iso, u1, -uu * uy); b2 = fmaf(s_iso, u2, -uu * uz);
    }
    const int ht = st.res_ht[k], ho = st.res_ho[k];
    float c0 = b0, c1 = b1, c2 = b2;
    if (!pos_loss) {
      if (dm.loss == DEXR_LOSS_DEXPILOT && k < dm.len_proj && flags[k]) {
        // projected pair t = eta e / (|e| + 1e-6), e the human vector: dt/de = eta / (|e| + eps) (I - e e^T / (|e| (|e| + eps)))
        float ex, ey, ez;
        if (by_kp) {
          ex = in.kp[3 * ht] - in.kp[3 * ho]; ey = in.kp[3 * ht + 1] - in.kp[3 * ho + 1]; ez = in.kp[3 * ht + 2] - in.kp[3 * ho + 2];
        } else {
          ex = in.ref[3 * k]; ey = in.ref[3 * k + 1]; ez = in.ref[3 * k + 2];
        }
        const float dist = sqrtf(fmaf(ex, ex, fmaf(ey, ey, ez * ez)));
        const float den = dist + 1e-6f;
        const float sc = (k < dm.len_s1 ? sv.prm.eta1 : sv.prm.eta2) / den;
        const float de = dist > 0.f ? fmaf(ex, b0, fmaf(ey, b1, ez * b2)) / (dist * den) : 0.f;
        c0 = sc * fmaf(-de, ex, b0); c1 = sc * fmaf(-de, ey, b1); c2 = sc * fmaf(-de, ez, b2);
      } else {
        c0 = sv.prm.scaling * b0; c1 = sv.prm.scaling * b1; c2 = sv.prm.scaling * b2;
      }
    }
    const float cl = l == 0 ? c0 : (l == 1 ? c1 : c2);
    if (by_kp) {
      if (l < 3) {  // keypoints shared by several residuals (the wrist) accumulate; lane c owns coordinate c
        kpacc[3 * ht + l] += cl;
        if (ho >= 0) kpacc[3 * ho + l] -= cl;
      }
    } else if (active && grad_ref && l < 3) {
      grad_ref[k * 3 + l] = out(cl);
    }
  }
  // ---- fixed joints: q_bar_c = -H_q[c, :] . M v (the anchor's a_bar = 2 norm_delta v is the driver's)
  float qbar = 0.f;
  if (fixedi >= 0)
    for (int i = 0; i < dof; ++i) qbar = fmaf(hq[i * NP + l], mvs[i], qbar);
  __syncwarp();
  return VjpLane{v, qbar, finite, bad};
}

// One frame of dexr_solve_vjp (see dexr.h): reads qpos, grad_qpos and the frame's inputs, writes the requested cotangents
// and the status.  `dm` is the kernel argument's, as in evaluate_frame.
template <int G>
__device__ __forceinline__ void vjp_frame(Solver<G, 0>& sv, const FrameInputs& in, const dexr_vjp_t& io, const Dims& dm,
                                          long long f, bool active) {
  const int l = sv.l;
  const bool isvar = sv.var >= 0;
  float x = 0.f, x0 = 0.f, gbar = 0.f;
  if (active && isvar) {
    x = io.qpos[f * dm.n_var + sv.var];
    x0 = io.last_qpos ? io.last_qpos[f * dm.n_var + sv.var] : x;
    gbar = io.grad_qpos[f * dm.n_var + sv.var];
  }
  const float nd = io.last_qpos ? sv.prm.norm_delta : 0.f;  // no anchor: no regulariser
  const VjpFront fr = vjp_front(sv, in, dm, x, x0, gbar, nd, io.projected ? io.projected + f * dm.len_proj : nullptr, active);
  const VjpLane r = vjp_tail(sv, in, dm, fr, gbar, io.grad_ref_value ? io.grad_ref_value + f * dm.n_res * 3 : nullptr, active);
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const bool by_kp = in.kp != nullptr;
  const float* const kpacc = sv.scf() + VjpScratch<G>::kKp;
  // outputs: NaN for a frame with a non-finite input, 0 for one whose free Hessian is not positive definite
  auto out = [&](float val) { return !r.finite ? __int_as_float(0x7fc00000) : (r.bad ? 0.f : val); };
  if (active) {
    if (isvar && io.grad_last_qpos) io.grad_last_qpos[f * dm.n_var + sv.var] = out(2.0f * nd * r.v);
    if (fixedi >= 0 && io.grad_fixed_qpos) io.grad_fixed_qpos[f * dm.n_fixed + fixedi] = out(-r.qbar);
    if (by_kp && io.grad_keypoints)
      for (int e = l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) io.grad_keypoints[f * 3 * DEXR_NUM_KEYPOINTS + e] = out(kpacc[e]);
    if (l == 0 && io.status_out) io.status_out[f] = !r.finite ? DEXR_STATUS_NONFINITE : (r.bad ? DEXR_STATUS_NOT_PD : 0);
  }
  __syncwarp();  // the group's next frame rewrites the scratch this one read
}

// ------------------------------------------------------------------------------------------------
// per-frame Jacobians of the solve (dexr_solve_jacobian): one front, then one tail per free variable
// ------------------------------------------------------------------------------------------------
// The argument checks of dexr_solve_jacobian that read the robot's table: nullptr, or what is wrong.  Host code shared by
// the library and the host emulation, as vjp_io_error.
inline const char* jacobian_io_error(const dexr_table_t& t, const dexr_jacobian_t& io, const dexr_params_t& prm) {
  if (!io.qpos) return "qpos is required";
  if ((io.keypoints != nullptr) == (io.ref_value != nullptr)) return "exactly one of keypoints / ref_value must be given";
  if (prm.preprocess != 0) return "raw-landmark pre-processing is not differentiated: params.preprocess must be 0";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  if (io.jac_keypoints && !io.keypoints) return "jac_keypoints needs the keypoints form";
  if (io.jac_ref_value && !io.ref_value) return "jac_ref_value needs the ref_value form";
  if (io.jac_last_qpos && !io.last_qpos) return "jac_last_qpos needs last_qpos";
  return nullptr;
}

// One frame of dexr_solve_jacobian (see dexr.h): vjp_front once, then for every variable i the row of cotangent e_i --
// vjp_tail with gbar = e_i where i is free, a zero row where it is active.  The warp's groups hold different frames but run
// the tail's collectives together: a row runs the tail when it is free in some group's frame, and a group whose own row i
// is active (or whose frame is bad) writes zeros (NaN for a non-finite frame) from it.  Row i of the frame is written from
// kpacc (keypoints), by the tail itself (ref_value), -qbar (fixed joints) and 2 norm_delta v (anchor).
template <int G>
__device__ __forceinline__ void jacobian_frame(Solver<G, 0>& sv, const FrameInputs& in, const dexr_jacobian_t& io,
                                               const Dims& dm, long long f, bool active) {
  const int l = sv.l, lane = sv.lane, n = dm.n_var;
  const bool isvar = sv.var >= 0;
  float x = 0.f, x0 = 0.f;
  if (active && isvar) {
    x = io.qpos[f * n + sv.var];
    x0 = io.last_qpos ? io.last_qpos[f * n + sv.var] : x;
  }
  const float nd = io.last_qpos ? sv.prm.norm_delta : 0.f;  // no anchor: no regulariser
  const VjpFront fr = vjp_front(sv, in, dm, x, x0, 0.f, nd, io.projected ? io.projected + f * dm.len_proj : nullptr, active);
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const bool by_kp = in.kp != nullptr;
  const float* const kpacc = sv.scf() + VjpScratch<G>::kKp;
  const float nan = __int_as_float(0x7fc00000);
  // a zero row for an active variable or a not-positive-definite frame, NaN for a frame with a non-finite input
  const float zero = fr.finite ? 0.f : nan;
  const bool good = active && fr.finite && !fr.bad;
  for (int i = 0; i < n; ++i) {
    const long long row = f * n + i;
    // row i of this group's frame needs the tail when variable i is free there; the warp runs it when some group needs it
    const unsigned need = __ballot_sync(0xffffffffu, good && fr.free_ && sv.var == i);
    const bool here = G == 32 ? need != 0u : ((need >> (lane & ~(G - 1))) & ((1u << (G & 31)) - 1u)) != 0u;
    float v = 0.f, qbar = 0.f;
    if (need != 0u) {  // (warp-uniform)
      const VjpLane r = vjp_tail(sv, in, dm, fr, sv.var == i ? 1.0f : 0.f,
                                 here && io.jac_ref_value ? io.jac_ref_value + row * dm.n_res * 3 : nullptr, active);
      v = r.v;
      qbar = r.qbar;
    }
    if (active) {
      if (isvar && io.jac_last_qpos) io.jac_last_qpos[row * n + sv.var] = here ? 2.0f * nd * v : zero;
      if (fixedi >= 0 && io.jac_fixed_qpos) io.jac_fixed_qpos[row * dm.n_fixed + fixedi] = here ? -qbar : zero;
      if (by_kp && io.jac_keypoints)
        for (int e = l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) io.jac_keypoints[row * 3 * DEXR_NUM_KEYPOINTS + e] = here ? kpacc[e] : zero;
      if (!here && !by_kp && io.jac_ref_value && l < 3)
        for (int k = 0; k < dm.n_res; ++k) io.jac_ref_value[row * dm.n_res * 3 + k * 3 + l] = zero;
    }
  }
  if (active && l == 0 && io.status_out) io.status_out[f] = !fr.finite ? DEXR_STATUS_NONFINITE : (fr.bad ? DEXR_STATUS_NOT_PD : 0);
  __syncwarp();  // the group's next frame rewrites the scratch this one read
}

// ------------------------------------------------------------------------------------------------
// backpropagation through the sequence solve (dexr_solve_sequences_vjp): the reverse-time recurrence of a stream
// ------------------------------------------------------------------------------------------------
// The argument checks of dexr_solve_sequences_vjp that read the robot's table or the parameters: nullptr, or what is wrong.
// Host code shared by the library and the host emulation, as vjp_io_error.
inline const char* seq_vjp_io_error(const dexr_table_t& t, const dexr_sequences_vjp_t& io, const dexr_params_t& prm) {
  if (prm.preprocess != 0) return "raw-landmark pre-processing is not differentiated: params.preprocess must be 0";
  if (!io.qpos) return "qpos (the tape of the forward call) is required";
  if (!io.last_qpos) return "last_qpos (the warm start before the forward call) is required";
  if (!io.keypoints) return "keypoints are required";
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  if (use_filter && !io.filter_init) return "the low-pass filter needs filter_init (as before the forward call)";
  if (t.loss == DEXR_LOSS_DEXPILOT && !io.projected) return "DexPilot needs the flag tape (projected)";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  return nullptr;
}

// One stream s of S, walked from its last frame to its first (dexr.h, dexr_solve_sequences_vjp): gy (the filter's cotangent,
// lane = joint) and c (the anchor cotangent flowing to the previous solution, lane = variable) stay in registers between
// frames; each frame runs vjp_front and vjp_tail at (x_t, clip(x_{t-1})) with gbar = M^T gq + c.  A group that is not `active` walks
// stream S - 1 and writes nothing.  `dm`, S and steps are the kernel argument's, as in solve_stream.
template <int G>
__device__ __forceinline__ void vjp_stream(Solver<G, 0>& sv, const dexr_sequences_vjp_t& io, const Dims& dm, const long long& S,
                                           const int& steps, long long s, bool active, bool use_filter) {
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l;
  const bool isvar = sv.var >= 0, isjoint = l < dm.dof;
  const long long sc = active ? s : S - 1;
  const float alpha = sv.prm.lp_alpha, nd = sv.prm.norm_delta;
  float gy = 0.f, c = 0.f;
  if (active && isjoint && io.grad_filter_state_out) gy = io.grad_filter_state_out[sc * dm.dof + l];
  if (active && isvar && io.grad_last_qpos_out) c = io.grad_last_qpos_out[sc * dm.n_var + sv.var];
  const bool finit = active && use_filter && io.filter_init[sc];
  for (int t = steps - 1; t >= 0; --t) {
    const long long fr = sc * steps + t;
    // dl/dq_t of this lane's joint: the output's cotangent, through the filter (y_t = y_{t-1} + alpha (q_t - y_{t-1}))
    float gq = (active && isjoint && io.grad_robot_qpos) ? io.grad_robot_qpos[fr * dm.dof + l] : 0.f;
    if (use_filter) {
      gy += gq;
      const bool init = t > 0 || finit;
      gq = init ? alpha * gy : gy;
      gy = init ? (1.0f - alpha) * gy : 0.f;
    }
    // gbar = M^T gq on the variables (mimic followers folded into their source, as in evaluate_frame) + the anchor cotangent
    float gbar = gq;
    if (dm.has_mimic) {
      const int gcount = st.group_count[l];
      float gx_ = 0.f;
#pragma unroll
      for (int k = 0; k < DEXR_MAX_GROUP; ++k) {
        const bool v = isvar && k < gcount;
        const float gv = gshfl<G>(gq, v ? st.group_lane[l][k] : l);
        if (v) gx_ = fmaf(st.group_mult[l][k], gv, gx_);
      }
      gbar = gx_;
    }
    gbar = isvar ? gbar + c : 0.f;
    // the point x_t and the anchor a_t = clip(x_{t-1}) the forward solved from
    float x = 0.f, xp = 0.f;
    if (active && isvar) {
      x = io.qpos[fr * dm.n_var + sv.var];
      xp = t > 0 ? io.qpos[(fr - 1) * dm.n_var + sv.var] : io.last_qpos[sc * dm.n_var + sv.var];
    }
    const float clo = st.clip_lo[l], chi = st.clip_hi[l];
    const float a = fminf(fmaxf(xp, clo), chi);
    const bool passes = xp >= clo && xp <= chi;  // the clip passes the anchor's cotangent (inclusive bounds, as torch.clamp)
    FrameInputs in;
    in.kp = io.keypoints + fr * (3 * DEXR_NUM_KEYPOINTS);
    in.ref = nullptr;
    in.fixed = dm.n_fixed > 0 ? io.fixed_qpos + fr * dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = nullptr;
    const VjpFront vf = vjp_front(sv, in, dm, x, a, gbar, nd, io.projected ? io.projected + fr * dm.len_proj : nullptr, active);
    const VjpLane r = vjp_tail(sv, in, dm, vf, gbar, nullptr, active);
    // outputs: NaN for a frame with a non-finite input (and, through c, for every earlier frame of the stream); v = 0 for
    // one whose free Hessian is not positive definite
    auto out = [&](float val) { return !r.finite ? __int_as_float(0x7fc00000) : val; };
    // the anchor's cotangent reaches x_{t-1} where the clip passes it; NaN stays NaN
    c = out(2.0f * nd * r.v) * (passes ? 1.0f : 0.f);
    if (active) {
      const int fixedi = st.fixed_index[l];
      const float* const kpacc = sv.scf() + VjpScratch<G>::kKp;
      if (fixedi >= 0 && io.grad_fixed_qpos) io.grad_fixed_qpos[fr * dm.n_fixed + fixedi] = out(gq - r.qbar);
      if (io.grad_keypoints)
        for (int e = l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) io.grad_keypoints[fr * 3 * DEXR_NUM_KEYPOINTS + e] = out(kpacc[e]);
      if (l == 0 && io.status_out) io.status_out[fr] = !r.finite ? DEXR_STATUS_NONFINITE : (r.bad ? DEXR_STATUS_NOT_PD : 0);
    }
    __syncwarp();  // the next frame rewrites the scratch this one read
  }
  if (active) {
    if (isvar && io.grad_last_qpos) io.grad_last_qpos[sc * dm.n_var + sv.var] = c;
    if (isjoint && io.grad_filter_state)  // (without a filter gy is still the incoming cotangent: the state passes through)
      io.grad_filter_state[sc * dm.dof + l] = gy;
  }
}

// ------------------------------------------------------------------------------------------------
// packed streams (dexr_solve_sequences_packed / _packed_vjp): streams of any lengths, frames laid end to end
// ------------------------------------------------------------------------------------------------
// The argument checks of the packed calls: nullptr, or what is wrong.  Host code shared by the library and the host
// emulation.  `tape` nullptr: the unrecorded forward.  offsets live on the device and are not read here.
inline const char* packed_io_error(const dexr_table_t& t, const dexr_sequences_t& io, const dexr_sequences_tape_t* tape,
                                   const dexr_params_t& prm, const int64_t* offsets, long long S, long long N) {
  if (S < 0 || N < 0 || N > INT32_MAX) return "bad sizes: num_streams and num_frames must be >= 0, num_frames <= INT32_MAX";
  if (!offsets) return "offsets (device [S+1]) are required";
  if (!io.keypoints || !io.last_qpos || !io.robot_qpos_out) return "keypoints, last_qpos, robot_qpos_out required";
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  if (use_filter && (!io.filter_state || !io.filter_init)) return "low-pass filter needs filter_state and filter_init";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  if (tape) {
    if (prm.preprocess != 0) return "raw-landmark pre-processing is not recorded: params.preprocess must be 0 with a tape";
    if (!tape->qpos) return "tape->qpos is required";
    if (t.loss == DEXR_LOSS_DEXPILOT && (!tape->projected || !io.projected))
      return "DexPilot: the flag tape needs tape->projected and io->projected";
  }
  return nullptr;
}

inline const char* packed_io_error(const dexr_table_t& t, const dexr_sequences_vjp_t& io, const dexr_params_t& prm,
                                   const int64_t* offsets, long long S, long long N) {
  if (S < 0 || N < 0 || N > INT32_MAX) return "bad sizes: num_streams and num_frames must be >= 0, num_frames <= INT32_MAX";
  if (!offsets) return "offsets (device [S+1]) are required";
  return seq_vjp_io_error(t, io, prm);
}

// Where the packed streams lie: offsets [S+1] into the N frames.
struct PackedLayout {
  const int64_t* offsets;
  long long S, N;
};

// Stream number s (-1: none) and frame range of stream i.  A malformed range reads as an empty stream, so no layout can
// make a kernel reach outside its buffers.
struct PackedStream {
  long long s, first;
  int len;
};

__device__ __forceinline__ PackedStream packed_stream(const PackedLayout& pk, long long i) {
  PackedStream r{-1, 0, 0};
  if (i < 0 || i >= pk.S) return r;
  r.s = i;
  const long long a = pk.offsets[i], b = pk.offsets[i + 1];
  if (a >= 0 && a <= b && b <= pk.N) {
    r.first = a;
    r.len = (int)(b - a);  // (N <= INT32_MAX)
  }
  return r;
}

// The longer of the warp's stream lengths: every group of a warp walks the time loop that long (warp-wide shuffles inside
// solve and vjp_front).
template <int G>
__device__ __forceinline__ int warp_steps(int len) {
  if constexpr (G == 16) {
    const int other = __shfl_xor_sync(0xffffffffu, len, 16);
    return other > len ? other : len;
  } else {
    return len;
  }
}

// solve_stream for one packed stream `ps` (ps.s < 0: none).  `works`: this group solves the stream (the owner, or the
// helping half-warp in duo mode); `writes`: it stores results and state.  The warp loops to the longer of its groups'
// lengths; a group past its end (or without a stream) solves a valid frame inactive -- its own last frame, or frame 0 --
// with writes off.  Its state is stored at its own last frame, so the extra frames change nothing it wrote.  Per frame the
// arithmetic is solve_stream's; a twin rather than a generalisation, which would move the machine code of the
// rectangular sequences kernels.
template <int G, int BW, bool REC>
__device__ __forceinline__ void solve_packed_stream(Solver<G, BW>& sv, const dexr_sequences_t& io, const Dims& dm,
                                                    const dexr_params_t& prm, const PackedStream& ps, bool works, bool writes,
                                                    float* kpbuf, bool use_filter, float* tape_qpos, uint8_t* tape_proj) {
  constexpr int KPL = (3 * DEXR_NUM_KEYPOINTS + G - 1) / G;
  const int l = sv.l;
  const int len = works && ps.s >= 0 ? ps.len : 0;
  const int steps = warp_steps<G>(len);
  if (steps == 0) return;
  const bool has = len > 0;
  writes = writes && has;
  const long long sc = has ? ps.s : 0, f0 = has ? ps.first : 0;
  const int tlast = has ? len - 1 : 0;
  float last = 0.f, fy = 0.f;
  int finit = 0;
  if (has && sv.var >= 0) last = io.last_qpos[sc * dm.n_var + sv.var];
  if (has && use_filter && l < dm.dof) fy = io.filter_state[sc * dm.dof + l];
  if (has && use_filter) finit = io.filter_init[sc];
  sv.lam_carry = (has && io.damping_state) ? io.damping_state[sc] : 0.f;
  const float* kp_stream = io.keypoints + f0 * (3 * DEXR_NUM_KEYPOINTS);
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
      const float* nxt = kp_stream + (long long)(t + 1 < tlast ? t + 1 : tlast) * (3 * DEXR_NUM_KEYPOINTS);
#pragma unroll
      for (int j = 0; j < KPL; ++j) {
        const int e = l + j * G;
        pre[j] = (e < 3 * DEXR_NUM_KEYPOINTS) ? nxt[e] : 0.f;
      }
    }
    __syncwarp();
    const bool act = t < len;
    const long long fr = f0 + (t < tlast ? t : tlast);
    FrameInputs in;
    in.kp = kpbuf;
    in.ref = nullptr;
    in.fixed = dm.n_fixed > 0 ? io.fixed_qpos + fr * dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = io.projected ? io.projected + sc * dm.len_proj : nullptr;
    sv.x = last;
    const int status = sv.solve(in, act);
    last = sv.x;
    const bool w = writes && act;
    if constexpr (REC) {
      if (w) {
        if (sv.var >= 0) tape_qpos[fr * dm.n_var + sv.var] = last;
        if (tape_proj && l < dm.len_proj) tape_proj[fr * dm.len_proj + l] = io.projected[sc * dm.len_proj + l];
      }
    }
    float out = sv.q;
    if (use_filter) {
      fy = finit ? fmaf(prm.lp_alpha, out - fy, fy) : out;
      finit = 1;
      out = fy;
    }
    if (w) {
      if (l < dm.dof) io.robot_qpos_out[fr * dm.dof + l] = out;
      if (l == 0 && io.status_out) io.status_out[fr] = status;
      if (t == tlast) {
        if (sv.var >= 0) io.last_qpos[sc * dm.n_var + sv.var] = last;
        if (use_filter && l < dm.dof) io.filter_state[sc * dm.dof + l] = fy;
        if (use_filter && l == 0) io.filter_init[sc] = (uint8_t)finit;
        if (io.damping_state && l == 0) io.damping_state[sc] = sv.lam_carry;
      }
    }
    __syncwarp();
  }
}

// vjp_stream for one packed stream `ps` (ps.s < 0: none), walked from its last frame to its first while the warp walks
// t = steps - 1 .. 0; frames past the group's end run inactive on a valid frame and leave gy and c as they are.  A
// stream of length 0 passes its state cotangents through.  Per frame the arithmetic is vjp_stream's.
template <int G>
__device__ __forceinline__ void vjp_packed_stream(Solver<G, 0>& sv, const dexr_sequences_vjp_t& io, const Dims& dm,
                                                  const PackedStream& ps, bool owner, bool use_filter) {
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l;
  const bool isvar = sv.var >= 0, isjoint = l < dm.dof;
  const bool valid = owner && ps.s >= 0;
  const int len = valid ? ps.len : 0;
  const int steps = warp_steps<G>(len);
  const long long sc = valid ? ps.s : 0, f0 = len > 0 ? ps.first : 0;
  const int tlast = len > 0 ? len - 1 : 0;
  const float alpha = sv.prm.lp_alpha, nd = sv.prm.norm_delta;
  float gy = 0.f, c = 0.f;
  if (valid && isjoint && io.grad_filter_state_out) gy = io.grad_filter_state_out[sc * dm.dof + l];
  if (valid && isvar && io.grad_last_qpos_out) c = io.grad_last_qpos_out[sc * dm.n_var + sv.var];
  const bool finit = valid && use_filter && io.filter_init[sc];
  for (int t = steps - 1; t >= 0; --t) {
    const bool act = t < len;
    const long long fr = f0 + (t < tlast ? t : tlast);
    float gq = (act && isjoint && io.grad_robot_qpos) ? io.grad_robot_qpos[fr * dm.dof + l] : 0.f;
    float gyn = gy;
    if (use_filter) {
      gyn += gq;
      const bool init = t > 0 || finit;
      gq = init ? alpha * gyn : gyn;
      gyn = init ? (1.0f - alpha) * gyn : 0.f;
    }
    float gbar = gq;
    if (dm.has_mimic) {
      const int gcount = st.group_count[l];
      float gx_ = 0.f;
#pragma unroll
      for (int k = 0; k < DEXR_MAX_GROUP; ++k) {
        const bool v = isvar && k < gcount;
        const float gv = gshfl<G>(gq, v ? st.group_lane[l][k] : l);
        if (v) gx_ = fmaf(st.group_mult[l][k], gv, gx_);
      }
      gbar = gx_;
    }
    gbar = isvar ? gbar + c : 0.f;
    float x = 0.f, xp = 0.f;
    if (act && isvar) {
      x = io.qpos[fr * dm.n_var + sv.var];
      xp = t > 0 ? io.qpos[(fr - 1) * dm.n_var + sv.var] : io.last_qpos[sc * dm.n_var + sv.var];
    }
    const float clo = st.clip_lo[l], chi = st.clip_hi[l];
    const float a = fminf(fmaxf(xp, clo), chi);
    const bool passes = xp >= clo && xp <= chi;
    FrameInputs in;
    in.kp = io.keypoints + fr * (3 * DEXR_NUM_KEYPOINTS);
    in.ref = nullptr;
    in.fixed = dm.n_fixed > 0 ? io.fixed_qpos + fr * dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = nullptr;
    const VjpFront vf = vjp_front(sv, in, dm, x, a, gbar, nd, io.projected ? io.projected + fr * dm.len_proj : nullptr, act);
    const VjpLane r = vjp_tail(sv, in, dm, vf, gbar, nullptr, act);
    auto out = [&](float val) { return !r.finite ? __int_as_float(0x7fc00000) : val; };
    const float cn = out(2.0f * nd * r.v) * (passes ? 1.0f : 0.f);
    if (act) {
      gy = gyn;
      c = cn;
      const int fixedi = st.fixed_index[l];
      const float* const kpacc = sv.scf() + VjpScratch<G>::kKp;
      if (fixedi >= 0 && io.grad_fixed_qpos) io.grad_fixed_qpos[fr * dm.n_fixed + fixedi] = out(gq - r.qbar);
      if (io.grad_keypoints)
        for (int e = l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) io.grad_keypoints[fr * 3 * DEXR_NUM_KEYPOINTS + e] = out(kpacc[e]);
      if (l == 0 && io.status_out) io.status_out[fr] = !r.finite ? DEXR_STATUS_NONFINITE : (r.bad ? DEXR_STATUS_NOT_PD : 0);
    }
    __syncwarp();
  }
  if (valid) {
    if (isvar && io.grad_last_qpos) io.grad_last_qpos[sc * dm.n_var + sv.var] = c;
    if (isjoint && io.grad_filter_state) io.grad_filter_state[sc * dm.dof + l] = gy;
  }
}

// ------------------------------------------------------------------------------------------------
// offline smoothing of packed streams (dexr_smooth_sequences_packed): every frame of a stream solved jointly
// ------------------------------------------------------------------------------------------------
// F(X) = sum_t L_t(x_t) + w sum_{t>=1} |x_t - x_{t-1}|^2 + w |x_0 - a|^2 is minimised by a damped projected Newton method,
// one group of G lanes per stream (lane = joint, as in the VJP).  Its Hessian is block tridiagonal: D_t = M^T H_q M + 2 w k_t I
// (+ mu I, the damping) on the diagonal, -2 w I beside it.  One outer iteration is three sweeps along the clip:
//   forward   at x_t: targets (the DexPilot flag recurrence), FK, the data gradient and H_q (exact_grad_hq, as in the VJP),
//             the smoothness gradient, the active set (the solver's rule on the TOTAL gradient), then block Thomas:
//             S_t = D_t - (2w)^2 Z_{t-1} and y_t = -g_t + 2w Z_{t-1} y_{t-1} over the free variables of frame t, with
//             Z_t the inverse of S_t over its free variables and zero elsewhere (so the free sets of t-1 and t need no
//             further masking).  S_t is factorised (factor_rows) and inverted, one column per lane, into the workspace;
//   backward  delta_t = Z_t (y_t + 2w delta_{t+1}) and the trial clip(x_t + delta_t) to the widened bounds;
//   cost      sum over frames and lanes of (this lane's term of F_t at the trial) - (the same at x), F_t = L_t(x_t) +
//             w |x_t - x_{t-1}|^2: per-term differences, not a difference of two fp32 totals over hundreds of frames.
// A decrease is accepted (mu x 0.1), and so is a change within the fp32 resolution of F when the predicted decrease is
// too (kSmoothNoise); anything else is rejected (mu x 10).  A pivot <= 0 in the forward sweep restarts it at once, first with
// the Gauss-Newton model (H_q without the kinematic curvature, positive semi-definite: the positive-definite fallback of the
// frame solver), then with more damping.  The stream stops when the max |delta| of a trial falls to params.tol, or after
// params.max_iters accepted outer iterations.
// A missing frame (non-finite keypoint or fixed joint) keeps only its smoothness terms (H_q = 0, no data gradient).
//
// Workspace per frame (floats), lane-space vectors of G entries:
//   kZ  [G][G] Z_t; entry [k][c] is written and read back by lane c only (column c of the inverse, which lane c uses as its
//              row: Z_t is symmetric up to rounding), so the accesses are coalesced and never cross lanes
//   kY  [G]    y_t
//   kX  [2][G] the iterate and the trial (0 on lanes without a variable)
//   kV  [G]    this lane's term of F_t at the iterate
//   kG  [G]    the total gradient g_t on the free variables (0 elsewhere), for the predicted decrease
template <int G>
struct SmoothWs {
  static constexpr int kZ = 0;
  static constexpr int kY = G * G;
  static constexpr int kX = kY + G;
  static constexpr int kV = kX + 2 * G;
  static constexpr int kG = kV + G;
  static constexpr int kFloats = kG + G;
};

// The workspace of the acceleration-penalised smoother (dexr_smooth_sequences_packed_accel, DESIGN.md 3.16): SmoothWs<G>
// followed by
//   kE  [G][G] E_t, the dense coupling block between frames t and t+1 that the banded elimination leaves: entry [k][c]
//              (row k: frame t's joint, column c: frame t+1's) at k * G + c, written by lane c
template <int G>
struct SmoothAccWs : SmoothWs<G> {
  static constexpr int kE = SmoothWs<G>::kFloats;
  static constexpr int kFloats = kE + G * G;
};

template <int G, bool ACC>
struct SmoothWsOf { using type = SmoothWs<G>; };
template <int G>
struct SmoothWsOf<G, true> { using type = SmoothAccWs<G>; };

// Relative resolution of F in the smoother's acceptance test: a trial whose change of F, and whose predicted decrease
// -g.delta / 2, both lie within kSmoothNoise F is accepted.  Near the minimiser the decrease a Newton step brings along a
// flat direction (a joint the keypoints hardly determine) is far below what the fp32 terms resolve; rejecting it there
// would only raise the damping until the step fell below tol, short of the minimiser.
constexpr float kSmoothNoise = 1e-6f;
// Damping beyond which a stream stops (with DEXR_STATUS_MAXITER): its steps are far below any tolerance by then.
constexpr float kSmoothMuMax = 1e12f;

// Bytes of workspace a call on `num_frames` frames needs (dexr_smooth_workspace_bytes).
inline size_t smooth_workspace_bytes(const dexr_table_t& t, long long num_frames) {
  const int floats = eval_lanes(t) == 16 ? SmoothWs<16>::kFloats : SmoothWs<32>::kFloats;
  return num_frames > 0 ? (size_t)num_frames * (size_t)floats * sizeof(float) : 0;
}

// Bytes of workspace an acceleration-penalised call on `num_frames` frames needs (dexr_smooth_accel_workspace_bytes).
inline size_t smooth_accel_workspace_bytes(const dexr_table_t& t, long long num_frames) {
  const int floats = eval_lanes(t) == 16 ? SmoothAccWs<16>::kFloats : SmoothAccWs<32>::kFloats;
  return num_frames > 0 ? (size_t)num_frames * (size_t)floats * sizeof(float) : 0;
}

// The extra argument checks of the acceleration-penalised entry points (after smooth_io_error / smooth_vjp_io_error):
// nullptr, or what is wrong.
inline const char* smooth_accel_error(const dexr_table_t& t, float accel_weight, const void* workspace,
                                      size_t workspace_bytes, long long N) {
  if (!(accel_weight >= 0.f && accel_weight <= 3.0e38f)) return "accel_weight must be finite and >= 0";
  if (N > 0 && (!workspace || workspace_bytes < smooth_accel_workspace_bytes(t, N)))
    return "workspace smaller than dexr_smooth_accel_workspace_bytes(robot, num_frames)";
  return nullptr;
}

// The argument checks of dexr_smooth_sequences_packed: nullptr, or what is wrong.  Host code shared by the library and the
// host emulation.  offsets live on the device and are not read here.
inline const char* smooth_io_error(const dexr_table_t& t, const dexr_smooth_t& io, const dexr_params_t& prm,
                                   const int64_t* offsets, long long S, long long N) {
  if (S < 0 || N < 0 || N > INT32_MAX) return "bad sizes: num_streams and num_frames must be >= 0, num_frames <= INT32_MAX";
  if (!offsets) return "offsets (device [S+1]) are required";
  if (prm.preprocess != 0) return "raw landmarks are not smoothed: params.preprocess must be 0 (pre-process the keypoints first)";
  if (!io.keypoints || !io.qpos_init || !io.qpos_out) return "keypoints, qpos_init and qpos_out are required";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  if (!(io.smooth_weight < 0.f) && !(io.smooth_weight >= 0.f && io.smooth_weight <= 3.0e38f))
    return "smooth_weight must be finite (< 0: params.norm_delta)";
  if (N > 0 && (!io.workspace || io.workspace_bytes < smooth_workspace_bytes(t, N)))
    return "workspace smaller than dexr_smooth_workspace_bytes(robot, num_frames)";
  return nullptr;
}

// Whether frame fr has a non-finite keypoint coordinate or fixed joint (group-uniform; false for a group that is not `live`).
template <int G>
__device__ __forceinline__ bool smooth_missing(const Solver<G, 0>& sv, const dexr_smooth_t& io, const Dims& dm, long long fr,
                                               bool live) {
  bool bad = false;
  if (live) {
    const float* kp = io.keypoints + fr * (3 * DEXR_NUM_KEYPOINTS);
    for (int e = sv.l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) bad = bad || !isfinite(kp[e]);
    const int fixedi = Solver<G, 0>::ST().fixed_index[sv.l];
    if (fixedi >= 0) bad = bad || !isfinite(io.fixed_qpos[fr * dm.n_fixed + fixedi]);
  }
  return gany<G>(bad, sv.lane);
}

// Frame fr at the point x (this lane's variable; xp: the previous frame's, or the anchor, when `has_prev`): advances the
// group's DexPilot flags in the scratch by one step of the hysteresis recurrence, prepares the targets, runs FK and returns
// this lane's term of F_t -- residual l of L_t (none for a missing frame) plus w (x - xp)^2 on a variable lane (w is
// sv.prm.norm_delta, which the launch sets to the smoothing weight).
template <int G>
__device__ __forceinline__ float smooth_eval(Solver<G, 0>& sv, const dexr_smooth_t& io, const Dims& dm, long long fr, float x,
                                             float xp, bool has_prev, bool missing, bool live) {
  const int l = sv.l;
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const float qf = (live && fixedi >= 0) ? io.fixed_qpos[fr * dm.n_fixed + fixedi] : 0.f;
  sv.qfix = isfinite(qf) ? qf : 0.f;
  sv.x = x;
  sv.x0 = has_prev ? xp : x;
  FrameInputs in;
  in.kp = io.keypoints + fr * (3 * DEXR_NUM_KEYPOINTS);
  in.ref = nullptr;
  in.fixed = nullptr;
  in.last = nullptr;
  in.projected = dm.len_proj > 0 ? reinterpret_cast<uint8_t*>(sv.scf() + VjpScratch<G>::kFlags) : nullptr;
  sv.prepare_targets(in, live);
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
  sv.cost(0, x);
  const float dx = x - sv.x0;
  const float reg = sv.var >= 0 ? fmaf(sv.prm.norm_delta * dx, dx, 0.f) : 0.f;
  return missing ? reg : sv.cost_lane;
}

// The group's DexPilot flags at the start of stream sc (nullptr: all false), into the scratch copy the sweeps advance.
template <int G>
__device__ __forceinline__ void smooth_reset_flags(const Solver<G, 0>& sv, const dexr_smooth_t& io, const Dims& dm, long long sc,
                                                   bool has) {
  uint8_t* const flags = reinterpret_cast<uint8_t*>(sv.scf() + VjpScratch<G>::kFlags);
  if (sv.l < dm.len_proj) flags[sv.l] = (has && io.projected) ? io.projected[sc * dm.len_proj + sv.l] : (uint8_t)0;
  __syncwarp();
}

// The acceleration-penalised smoother's coefficients at frame t of a stream of `len` frames (DESIGN.md 3.16): the triples
// (s-1, s, s+1) of F_c have centres s in [anchor ? 0 : 1, len - 2], the clipped anchor standing in for frame -1.  Frame t is
// the right end of the triple centred at t-1 (`right`), the centre of the one at t (`centre`) and the left end of the one at
// t+1 (`left`).  Group-uniform.
struct AccTerms {
  bool right, centre, left;
  __device__ __forceinline__ AccTerms(int t, int len, bool anchor)
      : right(t >= 2 || (t == 1 && anchor)), centre((t >= 1 || anchor) && t + 1 < len), left(t + 2 < len) {}
  // m_t: the sum of the squared coefficients (1, -2, 1) of frame t over its triples
  __device__ __forceinline__ float diag() const { return (right ? 1.f : 0.f) + (centre ? 4.f : 0.f) + (left ? 1.f : 0.f); }
  // the number of triples that hold both t and t+1
  __device__ __forceinline__ float pair() const { return (centre ? 1.f : 0.f) + (left ? 1.f : 0.f); }
  // d/dx_t of c times the triples' squares, from x_{t-2} .. x_{t+2} (x_{-1}: the anchor; entries of absent frames unused)
  __device__ __forceinline__ float grad(float c, float xp2, float xp, float x, float xn, float xn2) const {
    const float sr = x - 2.f * xp + xp2, sc = xn - 2.f * x + xp, sl = xn2 - 2.f * xn + x;
    return 2.f * c * ((right ? sr : 0.f) - (centre ? 2.f * sc : 0.f) + (left ? sl : 0.f));
  }
  // F_t's share of c times the triples' squares: the triple centred at t-1
  __device__ __forceinline__ float cost(float c, float xp2, float xp, float x) const {
    const float sr = x - 2.f * xp + xp2;
    return right ? c * sr * sr : 0.f;
  }
};

// The pre-anchor of a fixed-lag window solve with the acceleration penalty (smooth_packed_stream<G, true, true>,
// dexr_fixed_lag_step_accel, DESIGN.md 3.17).  Its state travels in io.cost_out, which a window solve leaves NULL (it
// writes no cost), as c travels in io.smooth_weight: a parameter of its own changes the code of the instantiations without
// it.  Read at each use rather than held in registers across the solve.
__device__ __forceinline__ const dexr_fixed_lag_accel_t* pre_anchor_state(const dexr_smooth_t& io) {
  return reinterpret_cast<const dexr_fixed_lag_accel_t*>(io.cost_out);
}
// Whether stream s has a pre-anchor (has_prev[s] non-zero; group-uniform).
__device__ __forceinline__ bool pre_anchor_on(const dexr_smooth_t& io, long long s, bool has) {
  return has && pre_anchor_state(io)->has_prev[s] != 0;
}
// The residual x - 2 clip(a) + clip(p) of the triple (p, a, x_0) on this var lane (`a`: its clip(a)); the stream has a
// pre-anchor.
template <int G>
__device__ __forceinline__ float pre_anchor_res(const Solver<G, 0>& sv, const dexr_smooth_t& io, long long s, int n, float a,
                                                float x) {
  const SharedTable& st = Solver<G, 0>::ST();
  const float p = fminf(fmaxf(pre_anchor_state(io)->prev_qpos[s * n + sv.var], st.clip_lo[sv.l]), st.clip_hi[sv.l]);
  return x - 2.f * a + p;
}

// The pre-anchor of a fixed-lag window VJP (smooth_vjp_packed_stream<G, true, true>, dexr_fixed_lag_step_accel_vjp, DESIGN.md
// 3.18).  The window view runs packed stream sc = 2 s only, so row sc + 1 of io.last_qpos holds its pre-anchor (raw) and row
// sc + 1 of io.grad_last_qpos takes its cotangent; the flags travel in io.workspace_bytes, which the kernel never reads (the
// device address of an int32 per packed stream), as the forward's pre-anchor state travels in io.cost_out.  Read at each use.
__device__ __forceinline__ bool pre_anchor_vjp_on(const dexr_smooth_vjp_t& io, long long sc, bool has) {
  return has && reinterpret_cast<const int32_t*>(io.workspace_bytes)[sc] != 0;
}
// pre_anchor_res for the window VJP (`a`: this lane's clip(a)).
template <int G>
__device__ __forceinline__ float pre_anchor_vjp_res(const Solver<G, 0>& sv, const dexr_smooth_vjp_t& io, long long sc, int n,
                                                    float a, float x) {
  const SharedTable& st = Solver<G, 0>::ST();
  const float p = fminf(fmaxf(io.last_qpos[(sc + 1) * n + sv.var], st.clip_lo[sv.l]), st.clip_hi[sv.l]);
  return x - 2.f * a + p;
}

// The banded block elimination's share of frame t (ACC), between fold_free_block and factor_rows: with the dense coupling
// E_{t-1} between frames t-1 and t and P = Z_{t-1} E_{t-1} (column per lane, in the kH area),
//   S_t = D_t - E_{t-1}^T P - c2^2 Z_{t-2},   y_t = y - P^T y_{t-1} - c2 Z_{t-2} y_{t-2},   E_t = b I - c1 P^T
// where b is the Hessian's scalar block between t and t+1, c1 the one between t-1 and t+1 and c2 the one between t-2 and t.
// `wt`: frame t's workspace (frames t-1 and t-2 before it; read only while `live`, which holds for them whenever it holds for
// t); `yp1`: this lane's y_{t-1} (y_{t-2} is read back from the workspace).  Z_{t-1}, Z_{t-2} are zero off their free
// variables, and the caller's A and y are only touched on frame t's, so the elimination is that of the free subproblem.
// E_t goes to the workspace; returns y_t.
template <int G, class W>
__device__ __forceinline__ float accel_eliminate(const Solver<G, 0>& sv, int dof, float* A, float* wt, int t, bool live,
                                                 bool free_, unsigned fmask, float y, float yp1, float b, float c1, float c2) {
  constexpr int NP = G;
  const int l = sv.l;
  const bool joint = l < dof;
  float* const P = sv.scf() + VjpScratch<G>::kH;
  const float* const zp = wt - W::kFloats + W::kZ;
  const float* const ep = wt - W::kFloats + W::kE;
  __syncwarp();  // fold_free_block has read H_q from the kH area (other lanes' columns, with mimic joints)
  if (t > 0) {  // (warp-uniform)
    for (int i = 0; i < dof; ++i) {
      float s = 0.f;
      if (live && joint)
        for (int k = 0; k < dof; ++k) s = fmaf(zp[i * G + k], ep[k * G + l], s);
      P[i * NP + l] = s;
    }
    __syncwarp();
    float py = 0.f;
    for (int k = 0; k < dof; ++k) py = fmaf(P[k * NP + l], gshfl<G>(yp1, k), py);
    if (free_) {
      y -= py;
      for (int c = 0; c < dof; ++c) {
        if (!((fmask >> c) & 1u)) continue;
        float s = 0.f;
        for (int k = 0; k < dof; ++k) s = fmaf(ep[k * G + l], P[k * NP + c], s);
        A[l * (NP + 1) + c] -= s;
      }
    }
  }
  if (t > 1) {  // (warp-uniform)
    const float* const zq = zp - W::kFloats;
    const float yp2 = live ? zq[W::kY - W::kZ + l] : 0.f;
    float zy = 0.f;
    for (int c = 0; c < dof; ++c) {
      const float z = live ? zq[c * G + l] : 0.f;
      zy = fmaf(z, gshfl<G>(yp2, c), zy);
      if (free_ && ((fmask >> c) & 1u)) A[l * (NP + 1) + c] = fmaf(-c2 * c2, z, A[l * (NP + 1) + c]);
    }
    if (free_) y = fmaf(-c2, zy, y);
  }
  if (live)
    for (int k = 0; k < dof; ++k) wt[W::kE + k * G + l] = (k == l ? b : 0.f) - ((t > 0 && joint) ? c1 * P[l * NP + k] : 0.f);
  __syncwarp();  // the factorisation and the inverse rewrite A and the kH area
  return y;
}

// The banded back substitution's right-hand side at frame t (ACC): y_t - E_t d_{t+1} - c2 d_{t+2} on this lane (`d1`: this
// lane's entry of d_{t+1}; d_{t+2} is read back from slot D of frame t+2's workspace; `n1`, `n2`: whether those frames exist).
template <int G, class W, int D>
__device__ __forceinline__ float accel_back_rhs(const float* wt, int l, int dof, bool live, bool n1, bool n2, float d1,
                                                float c2) {
  float ed = 0.f;
  for (int k = 0; k < dof; ++k) ed = fmaf((live && n1 && l < dof) ? wt[W::kE + l * G + k] : 0.f, gshfl<G>(d1, k), ed);
  return live ? wt[W::kY + l] - ed - (n2 ? c2 * wt[2 * W::kFloats + D + l] : 0.f) : 0.f;
}

// One packed stream `ps` (ps.s < 0: none) of dexr_smooth_sequences_packed; `owner`: this group runs the stream (the kernel
// gives a 16-lane warp's second group none).  The warp walks its groups' longer stream in every sweep and iterates until
// every group is done; a group that is done, or past its stream's end, runs its frames inactive with its writes off.  `ws`: the workspace,
// SmoothWs<G>::kFloats per frame.  `dm` and `prm` are the kernel argument's.
// ACC (dexr_smooth_sequences_packed_accel, DESIGN.md 3.16): F_c = F + c times the squared second differences of the
// stream (the anchor as frame -1), a block-pentadiagonal Hessian eliminated by accel_eliminate / accel_back_rhs in place of
// block Thomas, SmoothAccWs<G>::kFloats per frame; everything else as above.  c is io.smooth_weight: the launch has moved w
// into sv.prm.norm_delta, and c travels in the io rather than in a parameter of its own, which would change the code of the
// velocity-only instantiation.
// PRE (with ACC; dexr_fixed_lag_step_accel, DESIGN.md 3.17): stream s with has_prev[s] non-zero in the pre-anchor state
// (pre_anchor_state: io.cost_out, so no cost is written) adds the triple (clip(prev_qpos[s]), clip(a), x_0):
// c |x_0 - 2 clip(a) + clip(p)|^2 joins F_0, x_0's gradient and x_0's diagonal block (+2c); nothing off the diagonal
// changes.  A non-finite prev_qpos there is a non-finite start.
template <int G, bool ACC = false, bool PRE = false>
__device__ __forceinline__ void smooth_packed_stream(Solver<G, 0>& sv, const dexr_smooth_t& io, const Dims& dm,
                                                     const dexr_params_t& prm, const PackedStream& ps, bool owner, float* ws) {
  static_assert(ACC || !PRE, "the pre-anchor is a triple of the acceleration penalty");
  using W = typename SmoothWsOf<G, ACC>::type;
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, lane = sv.lane, dof = dm.dof, n = dm.n_var;
  const bool isvar = sv.var >= 0;
  const bool valid = owner && ps.s >= 0;
  const int len = valid ? ps.len : 0;
  const int steps = warp_steps<G>(len);
  if (steps == 0) return;
  const bool has = len > 0;
  const long long sc = has ? ps.s : 0, f0 = has ? ps.first : 0;
  const int tlast = has ? len - 1 : 0;
  float* const wsf = ws + f0 * W::kFloats;
  float* const A = sv.scf() + VjpScratch<G>::kA;
  float* const hq = sv.scf() + VjpScratch<G>::kH;
  const float w = sv.prm.norm_delta, w2 = 2.0f * w;
  const bool anchor = io.last_qpos != nullptr;

  // ---- the anchor and the starting trajectory (clipped to the widened bounds), both checked for finiteness
  bool nonfinite = false;
  float a = 0.f;
  if (has && isvar && anchor) {
    const float ar = io.last_qpos[sc * n + sv.var];
    nonfinite = !isfinite(ar);
    a = fminf(fmaxf(ar, st.clip_lo[l]), st.clip_hi[l]);
    if constexpr (PRE)
      if (pre_anchor_on(io, sc, has)) nonfinite = nonfinite || !isfinite(pre_anchor_state(io)->prev_qpos[sc * n + sv.var]);
  }
  for (int t = 0; t < len; ++t) {
    float x = 0.f;
    if (isvar) {
      const float v = io.qpos_init[(f0 + t) * n + sv.var];
      nonfinite = nonfinite || !isfinite(v);
      x = fminf(fmaxf(v, sv.lo), sv.hi);
    }
    wsf[t * W::kFloats + W::kX + l] = x;
  }
  nonfinite = gany<G>(nonfinite, lane);

  // ---- outer iterations (every counter and verdict below is group-uniform).  `exact`: the forward sweep uses the exact
  // Hessians; after an elimination that met a pivot <= 0 the sweep is repeated at the same damping with the Gauss-Newton
  // model (positive semi-definite, so the system is positive definite), then with ten times the damping.
  float mu = prm.lambda0, F = 0.f;
  int cur = 0, iters = 0, rejects = 0;
  bool done = !has || nonfinite, maxit = false, exact = true;
  while (__ballot_sync(0xffffffffu, !done) != 0u) {
    const bool act = !done;
    // forward sweep
    smooth_reset_flags(sv, io, dm, sc, has);
    bool failed = false;
    float fsum = 0.f, yprev = 0.f;
    for (int t = 0; t < steps; ++t) {
      const bool live = act && t < len;
      const int tc = t < tlast ? t : tlast;
      const long long fr = f0 + tc;
      float* const wt = wsf + tc * W::kFloats;
      const bool missing = smooth_missing(sv, io, dm, fr, live);
      const bool has_prev = t > 0 || anchor, has_next = t + 1 < len;
      // (frame tc of the group's stream, or frame 0 without one, is in the workspace; its neighbours only while `live`)
      const float x = wt[W::kX + cur * G + l];
      const float xp = (live && t > 0) ? wt[W::kX + cur * G + l - W::kFloats] : a;
      const float xn = (live && has_next) ? wt[W::kX + cur * G + l + W::kFloats] : 0.f;
      const float v = smooth_eval(sv, io, dm, fr, x, xp, has_prev, missing, live);
      if constexpr (ACC) {  // with the triples' share of F_t
        const float xp2 = (live && t > 1) ? wt[W::kX + cur * G + l - 2 * W::kFloats] : a;
        float va = isvar ? v + AccTerms(t, len, anchor).cost(io.smooth_weight, xp2, xp, x) : v;
        if constexpr (PRE)
          if (t == 0 && isvar && pre_anchor_on(io, sc, has)) {  // the triple (p, a, x_0)
            const float r = pre_anchor_res(sv, io, sc, n, a, x);
            va += io.smooth_weight * r * r;
          }
        if (live) {
          wt[W::kV + l] = va;
          fsum += va;
        }
      } else if (live) {
        wt[W::kV + l] = v;
        fsum += v;
      }
      float g = exact_grad_hq(sv, dm, exact);
      if (missing) {
        g = 0.f;
#pragma unroll
        for (int i = 0; i < NP; ++i) hq[i * NP + l] = 0.f;
      }
      g = isvar ? g + (has_prev ? w2 * (x - xp) : 0.f) + (has_next ? w2 * (x - xn) : 0.f) : 0.f;
      if constexpr (ACC) {  // the triples' share of g_t
        const AccTerms at(t, len, anchor);
        const float xp2 = (live && t > 1) ? wt[W::kX + cur * G + l - 2 * W::kFloats] : a;
        const float xn2 = (live && at.left) ? wt[W::kX + cur * G + l + 2 * W::kFloats] : 0.f;
        if (isvar) g += at.grad(io.smooth_weight, xp2, xp, x, xn, xn2);
        if constexpr (PRE)
          if (t == 0 && isvar && pre_anchor_on(io, sc, has))  // the triple (p, a, x_0)
            g += 2.f * io.smooth_weight * pre_anchor_res(sv, io, sc, n, a, x);
      }
      const bool at_bound = isvar && ((x <= sv.lo && g > -kGradNoise) || (x >= sv.hi && g < kGradNoise));
      const bool free_ = live && isvar && !at_bound;
      const unsigned fmask = gballot<G>(free_, lane);
      __syncwarp();
      if constexpr (ACC)
        fold_free_block(sv, dm, A, free_, fmask, fmaf(2.f * io.smooth_weight, AccTerms(t, len, anchor).diag(),
                                                      fmaf(w2, (float)((has_prev ? 1 : 0) + (has_next ? 1 : 0)), mu)));
      else
        fold_free_block(sv, dm, A, free_, fmask, fmaf(w2, (float)((has_prev ? 1 : 0) + (has_next ? 1 : 0)), mu));
      if constexpr (PRE)
        if (t == 0 && free_ && pre_anchor_on(io, sc, has))  // the triple (p, a, x_0): +2c on x_0's diagonal (row l: this lane's)
          A[l * (NP + 1) + l] += 2.f * io.smooth_weight;
      float y = free_ ? -g : 0.f;
      if constexpr (ACC)
        y = accel_eliminate<G, W>(sv, dof, A, wt, t, live, free_, fmask, y, yprev,
                                  -fmaf(4.f * io.smooth_weight, AccTerms(t, len, anchor).pair(), w2),
                                  (t >= 1 && has_next) ? 2.f * io.smooth_weight : 0.f, 2.f * io.smooth_weight);
      if (!ACC && t > 0) {  // (warp-uniform) the Schur complement of frame t - 1: Z_{t-1} is zero off its free variables
        const float* zp = wt - W::kFloats + W::kZ;
        float zy = 0.f;
        for (int c = 0; c < dof; ++c) {
          const float z = live ? zp[c * G + l] : 0.f;
          zy = fmaf(z, gshfl<G>(yprev, c), zy);
          if (free_ && ((fmask >> c) & 1u)) A[l * (NP + 1) + c] = fmaf(-w2 * w2, z, A[l * (NP + 1) + c]);
        }
        if (free_) y = fmaf(w2, zy, y);
      }
      const bool bad = factor_rows<G>(A, dof, l);
      __syncwarp();
      failed = failed || (live && bad);
      // Z_t, column l: L L^T z = e_l by forward and back substitution over the factor, z in the kH area (H_q is folded
      // into A by now), entry k of lane l at hq[k * NP + l]: the factor's reads are broadcasts, z's conflict-free
      for (int k = 0; k < dof; ++k) {
        float s = k == l ? 1.0f : 0.f;
        for (int i = 0; i < k; ++i) s = fmaf(-A[k * (NP + 1) + i], hq[i * NP + l], s);
        hq[k * NP + l] = s / A[k * (NP + 1) + k];
      }
      for (int k = dof - 1; k >= 0; --k) {
        float s = hq[k * NP + l];
        for (int i = k + 1; i < dof; ++i) s = fmaf(-A[i * (NP + 1) + k], hq[i * NP + l], s);
        s = s / A[k * (NP + 1) + k];
        hq[k * NP + l] = s;
        if (live) wt[W::kZ + k * G + l] = (free_ && ((fmask >> k) & 1u)) ? s : 0.f;
      }
      if (live) {
        wt[W::kY + l] = y;
        wt[W::kG + l] = free_ ? g : 0.f;
      }
      yprev = y;
      __syncwarp();  // the next frame rewrites the scratch this one read
    }
    const float Fold = gsum<G>(fsum);
    if (act) F = Fold;
    const bool go = act && !failed;
    if (act && failed) {  // restart the forward sweep: no trial, no outer iteration
      if (exact) exact = false;
      else mu *= kLamUp;
      if (rejects < 127) ++rejects;
      if (!(mu <= kSmoothMuMax)) done = maxit = true;
    }
    if (__ballot_sync(0xffffffffu, go) == 0u) continue;  // (warp-uniform) no group has a trial to evaluate
    // backward sweep: the step and the trial
    float dn = 0.f, smax = 0.f, gd = 0.f;
    for (int t = steps - 1; t >= 0; --t) {
      const bool live = go && t < len;
      const int tc = t < tlast ? t : tlast;
      float* const wt = wsf + tc * W::kFloats;
      float r;
      if constexpr (ACC)
        r = accel_back_rhs<G, W, W::kY>(wt, l, dof, live, t + 1 < len, t + 2 < len, dn, 2.f * io.smooth_weight);
      else r = live ? wt[W::kY + l] + (t + 1 < len ? w2 * dn : 0.f) : 0.f;
      float d = 0.f;
      for (int c = 0; c < dof; ++c) d = fmaf(live ? wt[W::kZ + c * G + l] : 0.f, gshfl<G>(r, c), d);
      if (live) {
        const float x = wt[W::kX + cur * G + l];
        wt[W::kX + (cur ^ 1) * G + l] = isvar ? fminf(fmaxf(x + d, sv.lo), sv.hi) : 0.f;
        smax = fmaxf(smax, fabsf(d));
        gd = fmaf(wt[W::kG + l], d, gd);
        if constexpr (ACC) wt[W::kY + l] = d;  // (y_t is used up: d_t for frame t-2's right-hand side)
        dn = d;
      }
    }
    smax = gmax<G>(smax);
    const float pred = -0.5f * gsum<G>(gd);
    // cost sweep: per-term differences of F_t at the trial and at x
    smooth_reset_flags(sv, io, dm, sc, has);
    float dsum = 0.f, fnew = 0.f;
    for (int t = 0; t < steps; ++t) {
      const bool live = go && t < len;
      const int tc = t < tlast ? t : tlast;
      const long long fr = f0 + tc;
      float* const wt = wsf + tc * W::kFloats;
      const bool missing = smooth_missing(sv, io, dm, fr, live);
      const float x = wt[W::kX + (cur ^ 1) * G + l];
      const float xp = (live && t > 0) ? wt[W::kX + (cur ^ 1) * G + l - W::kFloats] : a;
      const float v = smooth_eval(sv, io, dm, fr, x, xp, t > 0 || anchor, missing, live);
      if constexpr (ACC) {  // with the triples' share of F_t
        const float xp2 = (live && t > 1) ? wt[W::kX + (cur ^ 1) * G + l - 2 * W::kFloats] : a;
        float va = isvar ? v + AccTerms(t, len, anchor).cost(io.smooth_weight, xp2, xp, x) : v;
        if constexpr (PRE)
          if (t == 0 && isvar && pre_anchor_on(io, sc, has)) {  // the triple (p, a, x_0)
            const float r = pre_anchor_res(sv, io, sc, n, a, x);
            va += io.smooth_weight * r * r;
          }
        if (live) {
          dsum += va - wt[W::kV + l];
          fnew += va;
        }
      } else if (live) {
        dsum += v - wt[W::kV + l];
        fnew += v;
      }
      __syncwarp();
    }
    const float dF = gsum<G>(dsum), Fnew = gsum<G>(fnew);
    if (go) {
      if (dF < 0.f || (dF <= kSmoothNoise * Fold && pred <= kSmoothNoise * Fold)) {
        cur ^= 1;
        ++iters;
        mu = fmaxf(mu * kLamDown, kLamMin);
        F = Fnew;
      } else {
        mu *= kLamUp;
        if (rejects < 127) ++rejects;
      }
      exact = true;
      done = smax <= prm.tol;
      if (!done && (iters >= prm.max_iters || !(mu <= kSmoothMuMax))) done = maxit = true;
    }
  }

  // ---- outputs: the answer (qpos_init as given for a non-finite start), its scatter + mimic, the status, the cost
  const int base_status = nonfinite ? DEXR_STATUS_NONFINITE
                                    : ((iters & 0xffff) | (rejects << 16) | (maxit ? DEXR_STATUS_MAXITER : 0));
  const int fixedi = st.fixed_index[l];
  for (int t = 0; t < steps; ++t) {
    const bool live = has && t < len;
    const int tc = t < tlast ? t : tlast;
    const long long fr = f0 + tc;
    const bool missing = smooth_missing(sv, io, dm, fr, live && !nonfinite);
    float x = 0.f;
    if (live && isvar) x = nonfinite ? io.qpos_init[fr * n + sv.var] : wsf[tc * W::kFloats + W::kX + cur * G + l];
    sv.qfix = (live && fixedi >= 0) ? io.fixed_qpos[fr * dm.n_fixed + fixedi] : 0.f;
    const float q = sv.compose_q(x);
    if (live) {
      if (isvar) io.qpos_out[fr * n + sv.var] = x;
      if (io.robot_qpos_out && l < dof) io.robot_qpos_out[fr * dof + l] = q;
      if (io.status_out && l == 0) io.status_out[fr] = base_status | (missing ? DEXR_STATUS_MISSING : 0);
    }
  }
  if constexpr (!PRE)
    if (has && io.cost_out && l == 0) io.cost_out[sc] = nonfinite ? __int_as_float(0x7fc00000) : F;
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// backpropagation through the offline smoother (dexr_smooth_sequences_packed_vjp): one linear solve per stream
// ------------------------------------------------------------------------------------------------
// The argument checks of dexr_smooth_sequences_packed_vjp: nullptr, or what is wrong.  Host code shared by the library and
// the host emulation.  offsets live on the device and are not read here.
inline const char* smooth_vjp_io_error(const dexr_table_t& t, const dexr_smooth_vjp_t& io, const dexr_params_t& prm,
                                       const int64_t* offsets, long long S, long long N) {
  if (S < 0 || N < 0 || N > INT32_MAX) return "bad sizes: num_streams and num_frames must be >= 0, num_frames <= INT32_MAX";
  if (!offsets) return "offsets (device [S+1]) are required";
  if (prm.preprocess != 0) return "raw landmarks are not differentiated: params.preprocess must be 0 (pre-process the keypoints first)";
  if (!io.keypoints || !io.qpos || !io.grad_keypoints) return "keypoints, qpos and grad_keypoints are required";
  if (t.n_fixed > 0 && !io.fixed_qpos) return "the robot has fixed joints but fixed_qpos is NULL";
  if (io.grad_last_qpos && !io.last_qpos) return "grad_last_qpos needs last_qpos";
  if (!(io.smooth_weight < 0.f) && !(io.smooth_weight >= 0.f && io.smooth_weight <= 3.0e38f))
    return "smooth_weight must be finite (< 0: params.norm_delta)";
  if (N > 0 && (!io.workspace || io.workspace_bytes < smooth_workspace_bytes(t, N)))
    return "workspace smaller than dexr_smooth_workspace_bytes(robot, num_frames)";
  return nullptr;
}

// Packed stream `si` of `pk` (none when out of range) of dexr_smooth_sequences_packed_vjp (see dexr.h for the math); `owner`
// as in smooth_packed_stream.  Three sweeps along the clip, every frame at the given point X*:
//   forward   targets (the DexPilot flag recurrence), FK, H_q and the data gradient (smooth_eval, exact_grad_hq: the
//             smoother's own forward sweep with mu = 0, the exact model only), the active set on the total gradient, then
//             block Thomas: S_t = D_t - (2w)^2 Z_{t-1}, y_t = G_t + 2w Z_{t-1} y_{t-1}; Z_t and y_t into the workspace;
//   backward  v_t = Z_t (y_t + 2w v_{t+1}) into the workspace (the smoother's kX slot);
//   cotangent the frame again (targets, FK, H_q), then vjp_tail's target pass and fixed-joint term with v_t.
// The stream's NONFINITE and NOT_PD verdicts are known after the forward sweep and select every output.  `dm` and `ws` as in
// smooth_packed_stream; sv.prm.norm_delta holds w.
// ACC (dexr_smooth_sequences_packed_accel_vjp): the exact block-pentadiagonal Hessian of F_c (c = io.smooth_weight, as in
// smooth_packed_stream<G, true>), eliminated as the forward eliminates it with mu = 0; the anchor's cotangent gains
// 4c v_0 - 2c v_1 when the stream has a second frame.
// PRE (with ACC; dexr_fixed_lag_step_accel_vjp, DESIGN.md 3.18): a stream with a pre-anchor (pre_anchor_vjp_on) has the
// forward's triple (clip(p), clip(a), x_0): its share of g_0, +2c on x_0's diagonal block, a non-finite p as a non-finite
// stream, 4c v_0 more in the anchor's cotangent (after the terms above) and -2c v_0 as p's cotangent where the clip passes
// p (0 without a pre-anchor).
template <int G, bool ACC = false, bool PRE = false>
__device__ __forceinline__ void smooth_vjp_packed_stream(Solver<G, 0>& sv, const dexr_smooth_vjp_t& io, const Dims& dm,
                                                         const PackedLayout& pk, long long si, bool owner) {
  static_assert(ACC || !PRE, "the pre-anchor is a triple of the acceleration penalty");
  using W = typename SmoothWsOf<G, ACC>::type;
  constexpr int NP = G;
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, lane = sv.lane, dof = dm.dof, n = dm.n_var;
  const bool isvar = sv.var >= 0, isjoint = l < dof;
  const PackedStream ps = packed_stream(pk, si);
  const bool valid = owner && ps.s >= 0;
  const int len = valid ? ps.len : 0;
  const int steps = warp_steps<G>(len);
  const bool has = len > 0;
  const long long sc = si;  // (read only where `valid` holds: the caller's loop index, no register of its own)
  const int f0 = has ? (int)ps.first : 0;  // (num_frames <= INT32_MAX: 32 bits, one register fewer)
  const int tlast = has ? len - 1 : 0;
  // (the workspace is addressed from io.workspace per frame: a kernel argument, so no register holds its base)
  float* const A = sv.scf() + VjpScratch<G>::kA;
  float* const hq = sv.scf() + VjpScratch<G>::kH;
  const float w = sv.prm.norm_delta, w2 = 2.0f * w;
  const bool anchor = io.last_qpos != nullptr;
  // the forward's view of the inputs, for the smoother's frame helpers
  dexr_smooth_t fio{};
  fio.keypoints = io.keypoints;
  fio.fixed_qpos = io.fixed_qpos;
  fio.projected = io.projected;

  // G_t of this lane's variable at frame fr (0 off the variables), and `gq`, this lane's joint's grad_robot_qpos
  auto cotangent = [&](long long fr, bool live, float& gq) -> float {
    gq = (live && isjoint && io.grad_robot_qpos) ? io.grad_robot_qpos[fr * dof + l] : 0.f;
    float gb = gq;
    if (dm.has_mimic) {
      const int gcount = st.group_count[l];
      float gx_ = 0.f;
#pragma unroll
      for (int k = 0; k < DEXR_MAX_GROUP; ++k) {
        const bool v = isvar && k < gcount;
        const float gv = gshfl<G>(gq, v ? st.group_lane[l][k] : l);
        if (v) gx_ = fmaf(st.group_mult[l][k], gv, gx_);
      }
      gb = gx_;
    }
    if (live && isvar && io.grad_qpos) gb += io.grad_qpos[fr * n + sv.var];
    return isvar ? gb : 0.f;
  };

  // ---- the clipped anchor
  auto raw_anchor = [&]() { return (has && isvar && anchor) ? io.last_qpos[sc * n + sv.var] : 0.f; };
  auto clipped_anchor = [&]() { return fminf(fmaxf(raw_anchor(), st.clip_lo[l]), st.clip_hi[l]); };
  bool nonfinite = !isfinite(raw_anchor());
  if constexpr (PRE)
    if (isvar && pre_anchor_vjp_on(io, sc, has)) nonfinite = nonfinite || !isfinite(io.last_qpos[(sc + 1) * n + sv.var]);

  // ---- forward sweep: the elimination of H V = G.  G_t waits in the workspace's kG slot while the frame is evaluated, and
  // only the smoothness gradient of the neighbours stays in registers (the 16-lane kernel has 128 of them)
  smooth_reset_flags(sv, fio, dm, sc, has);
  bool bad = false;
  float yprev = 0.f;
  for (int t = 0; t < steps; ++t) {
    const bool live = t < len;
    const int tc = t < tlast ? t : tlast;
    const long long fr = (long long)(f0 + tc);
    float* const wt = static_cast<float*>(io.workspace) + (long long)(f0 + tc) * W::kFloats;
    const bool missing = smooth_missing(sv, fio, dm, fr, live);
    const bool has_prev = t > 0 || anchor, has_next = t + 1 < len;
    {
      float gq;
      const float gb = cotangent(fr, live, gq);
      nonfinite = nonfinite || !isfinite(gb) || !isfinite(gq);
      if (live) wt[W::kG + l] = gb;
    }
    float x = 0.f, xp = t > 0 ? 0.f : clipped_anchor(), xn = 0.f;
    if (live && isvar) {
      x = io.qpos[fr * n + sv.var];
      if (t > 0) xp = io.qpos[(fr - 1) * n + sv.var];
      if (has_next) xn = io.qpos[(fr + 1) * n + sv.var];
    }
    nonfinite = nonfinite || !isfinite(x);
    const float gs = (has_prev ? w2 * (x - xp) : 0.f) + (has_next ? w2 * (x - xn) : 0.f);
    smooth_eval(sv, fio, dm, fr, x, xp, has_prev, missing, live);
    float g = exact_grad_hq(sv, dm);
    if (missing) {
      g = 0.f;
#pragma unroll
      for (int i = 0; i < NP; ++i) hq[i * NP + l] = 0.f;
    }
    g = isvar ? g + gs : 0.f;
    if constexpr (ACC) {  // the triples' share of g_t (x_{-1}: the clipped anchor)
      const AccTerms at(t, len, anchor);
      float xp2 = t > 1 ? 0.f : clipped_anchor(), xn2 = 0.f, xn_ = 0.f;
      if (live && isvar) {
        if (t > 1) xp2 = io.qpos[(fr - 2) * n + sv.var];
        if (has_next) xn_ = io.qpos[(fr + 1) * n + sv.var];
        if (at.left) xn2 = io.qpos[(fr + 2) * n + sv.var];
      }
      if (isvar) g += at.grad(io.smooth_weight, xp2, xp, x, xn_, xn2);
      if constexpr (PRE)
        if (t == 0 && isvar && pre_anchor_vjp_on(io, sc, has))  // the triple (p, a, x_0); xp is clip(a) at t = 0
          g += 2.f * io.smooth_weight * pre_anchor_vjp_res(sv, io, sc, n, xp, x);
    }
    const bool at_bound = isvar && ((x <= sv.lo && g > -kGradNoise) || (x >= sv.hi && g < kGradNoise));
    const bool free_ = live && isvar && !at_bound;
    const unsigned fmask = gballot<G>(free_, lane);
    __syncwarp();
    if constexpr (ACC)
      fold_free_block(sv, dm, A, free_, fmask, fmaf(2.f * io.smooth_weight, AccTerms(t, len, anchor).diag(),
                                                    w2 * (float)((has_prev ? 1 : 0) + (has_next ? 1 : 0))));
    else
      fold_free_block(sv, dm, A, free_, fmask, w2 * (float)((has_prev ? 1 : 0) + (has_next ? 1 : 0)));
    if constexpr (PRE)
      if (t == 0 && free_ && pre_anchor_vjp_on(io, sc, has))  // the triple (p, a, x_0): +2c on x_0's diagonal
        A[l * (NP + 1) + l] += 2.f * io.smooth_weight;
    float y = (free_ && live) ? wt[W::kG + l] : 0.f;
    if constexpr (ACC)
      y = accel_eliminate<G, W>(sv, dof, A, wt, t, live, free_, fmask, y, yprev,
                                -fmaf(4.f * io.smooth_weight, AccTerms(t, len, anchor).pair(), w2),
                                (t >= 1 && has_next) ? 2.f * io.smooth_weight : 0.f, 2.f * io.smooth_weight);
    if (!ACC && t > 0) {  // (warp-uniform) the Schur complement of frame t - 1: Z_{t-1} is zero off its free variables
      const float* zp = wt - W::kFloats + W::kZ;
      float zy = 0.f;
      for (int c = 0; c < dof; ++c) {
        const float z = live ? zp[c * G + l] : 0.f;
        zy = fmaf(z, gshfl<G>(yprev, c), zy);
        if (free_ && ((fmask >> c) & 1u)) A[l * (NP + 1) + c] = fmaf(-w2 * w2, z, A[l * (NP + 1) + c]);
      }
      if (free_) y = fmaf(w2, zy, y);
    }
    const bool pb = factor_rows<G>(A, dof, l);
    __syncwarp();
    bad = bad || (live && pb);
    // Z_t, column l, as in smooth_packed_stream (z in the kH area, H_q is folded into A by now)
    for (int k = 0; k < dof; ++k) {
      float s = k == l ? 1.0f : 0.f;
      for (int i = 0; i < k; ++i) s = fmaf(-A[k * (NP + 1) + i], hq[i * NP + l], s);
      hq[k * NP + l] = s / A[k * (NP + 1) + k];
    }
    for (int k = dof - 1; k >= 0; --k) {
      float s = hq[k * NP + l];
      for (int i = k + 1; i < dof; ++i) s = fmaf(-A[i * (NP + 1) + k], hq[i * NP + l], s);
      s = s / A[k * (NP + 1) + k];
      hq[k * NP + l] = s;
      if (live) wt[W::kZ + k * G + l] = (free_ && ((fmask >> k) & 1u)) ? s : 0.f;
    }
    if (live) wt[W::kY + l] = y;
    yprev = y;
    __syncwarp();  // the next frame rewrites the scratch this one read
  }
  nonfinite = gany<G>(nonfinite, lane);

  // ---- backward sweep: v_t
  float vn = 0.f;
  for (int t = steps - 1; t >= 0; --t) {
    const bool live = t < len;
    const int tc = t < tlast ? t : tlast;
    float* const wt = static_cast<float*>(io.workspace) + (long long)(f0 + tc) * W::kFloats;
    float r;
    if constexpr (ACC)
      r = accel_back_rhs<G, W, W::kX>(wt, l, dof, live, t + 1 < len, t + 2 < len, vn, 2.f * io.smooth_weight);
    else r = live ? wt[W::kY + l] + (t + 1 < len ? w2 * vn : 0.f) : 0.f;
    float d = 0.f;
    for (int c = 0; c < dof; ++c) d = fmaf(live ? wt[W::kZ + c * G + l] : 0.f, gshfl<G>(r, c), d);
    if (live) {
      wt[W::kX + l] = d;
      vn = d;
    }
  }

  // ---- cotangent sweep: the target pass and the fixed-joint term of every frame with its v_t
  smooth_reset_flags(sv, fio, dm, sc, has);
  for (int t = 0; t < steps; ++t) {
    const bool live = t < len;
    const int tc = t < tlast ? t : tlast;
    const long long fr = (long long)(f0 + tc);
    const float* const wt = static_cast<float*>(io.workspace) + (long long)(f0 + tc) * W::kFloats;
    const bool missing = smooth_missing(sv, fio, dm, fr, live);
    float x = 0.f, xp = t > 0 ? 0.f : clipped_anchor();
    if (live && isvar) {
      x = io.qpos[fr * n + sv.var];
      if (t > 0) xp = io.qpos[(fr - 1) * n + sv.var];
    }
    smooth_eval(sv, fio, dm, fr, x, xp, t > 0 || anchor, missing, live);
    if (dm.n_fixed > 0) exact_grad_hq(sv, dm);  // (H_q into kH, for the fixed-joint term only; the gradient is not needed)
    FrameInputs in;
    in.kp = io.keypoints + fr * (3 * DEXR_NUM_KEYPOINTS);
    in.ref = nullptr;
    in.fixed = nullptr;
    in.last = nullptr;
    in.projected = nullptr;
    const float v = (live && isvar) ? wt[W::kX + l] : 0.f;
    const VjpLane r = vjp_tail<G, false>(sv, in, dm, VjpFront{isvar, true, false}, v, nullptr, live);
    // outputs: NaN for a non-finite stream, 0 for a NOT_PD one and on a missing frame
    auto out = [&](float val) { return nonfinite ? __int_as_float(0x7fc00000) : ((bad || missing) ? 0.f : val); };
    if (live) {
      const int fixedi = st.fixed_index[l];
      const float* const kpacc = sv.scf() + VjpScratch<G>::kKp;
      const int base_status = nonfinite ? DEXR_STATUS_NONFINITE : (bad ? DEXR_STATUS_NOT_PD : 0);
      const float gqd = (fixedi >= 0 && io.grad_robot_qpos) ? io.grad_robot_qpos[fr * dof + l] : 0.f;
      if (fixedi >= 0 && io.grad_fixed_qpos) io.grad_fixed_qpos[fr * dm.n_fixed + fixedi] = out(gqd - r.qbar);
      for (int e = l; e < 3 * DEXR_NUM_KEYPOINTS; e += G) io.grad_keypoints[fr * 3 * DEXR_NUM_KEYPOINTS + e] = out(kpacc[e]);
      if (l == 0 && io.status_out) io.status_out[fr] = base_status | (missing ? DEXR_STATUS_MISSING : 0);
    }
    __syncwarp();  // the next frame rewrites the scratch this one read
  }
  // ---- the anchor: 2 w v_0 where the clip passes it (an empty or malformed range: 0); v_0 is read back from the workspace
  // rather than held in a register through the cotangent sweep
  if (valid && isvar && io.grad_last_qpos) {
    const float ar = raw_anchor();
    const bool passes = ar >= st.clip_lo[l] && ar <= st.clip_hi[l];
    const float v0 = has ? static_cast<const float*>(io.workspace)[(long long)f0 * W::kFloats + W::kX + l] : 0.f;
    float ga = nonfinite ? __int_as_float(0x7fc00000) : ((bad || !passes) ? 0.f : w2 * v0);
    if constexpr (ACC) {  // g_0 and g_1 also depend on a through the triple (a, x_0, x_1)
      if (len > 1 && !nonfinite && !bad && passes) {
        const float v1 = static_cast<const float*>(io.workspace)[(long long)(f0 + 1) * W::kFloats + W::kX + l];
        ga = fmaf(2.f * io.smooth_weight, fmaf(2.f, v0, -v1), ga);
      }
    }
    if constexpr (PRE) {  // the triple (p, a, x_0): 4c v_0 more for a; -2c v_0 for p where the clip passes p
      float gp = 0.f;
      if (pre_anchor_vjp_on(io, sc, has)) {
        const float pr = io.last_qpos[(sc + 1) * n + sv.var];
        const bool ppass = pr >= st.clip_lo[l] && pr <= st.clip_hi[l];
        if (!nonfinite && !bad && passes) ga = fmaf(4.f * io.smooth_weight, v0, ga);
        gp = nonfinite ? __int_as_float(0x7fc00000) : ((bad || !ppass) ? 0.f : -2.f * io.smooth_weight * v0);
      }
      io.grad_last_qpos[(sc + 1) * n + sv.var] = gp;
    }
    io.grad_last_qpos[sc * n + sv.var] = has ? ga : 0.f;
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// fixed-lag smoothing of live streams (dexr_fixed_lag_step): each tick runs smooth_packed_stream on a window of the last
// L+1 frames held in the caller's state (see dexr.h for the semantics)
// ------------------------------------------------------------------------------------------------
// Bytes of workspace a call on S streams of lag L needs (dexr_fixed_lag_workspace_bytes): the smoother's for S (L+1) frames,
// then S (L+1) int32 status words (the window solve's, read back for the emitted frame).
inline size_t fixed_lag_workspace_bytes(const dexr_table_t& t, long long S, long long lag) {
  if (S <= 0 || lag < 0 || lag > DEXR_FIXED_LAG_MAX) return 0;
  const long long frames = S * (lag + 1);
  return smooth_workspace_bytes(t, frames) + (size_t)frames * sizeof(int32_t);
}

// Bytes of workspace an acceleration-penalised call needs (dexr_fixed_lag_accel_workspace_bytes): the accel smoother's for
// S (L+1) frames, then the S (L+1) status words.
inline size_t fixed_lag_accel_workspace_bytes(const dexr_table_t& t, long long S, long long lag) {
  if (S <= 0 || lag < 0 || lag > DEXR_FIXED_LAG_MAX) return 0;
  const long long frames = S * (lag + 1);
  return smooth_accel_workspace_bytes(t, frames) + (size_t)frames * sizeof(int32_t);
}

// Where the status words of a G-lane call's workspace start (ACC: after the accel smoother's frames).
template <int G, bool ACC = false>
inline int32_t* fixed_lag_status_words(const dexr_fixed_lag_t& io, long long S) {
  return reinterpret_cast<int32_t*>(static_cast<float*>(io.workspace) +
                                    S * (io.lag + 1) * SmoothWsOf<G, ACC>::type::kFloats);
}

// The argument checks of dexr_fixed_lag_step: nullptr, or what is wrong.  Host code shared by the library and the host
// emulation.  The per-tick inputs and outputs are required only when there are ticks.
inline const char* fixed_lag_io_error(const dexr_table_t& t, const dexr_fixed_lag_t& io, const dexr_params_t& prm,
                                      long long S, long long K) {
  if (S < 0 || K < 0 || K > INT32_MAX) return "bad sizes: num_streams and num_ticks must be >= 0, num_ticks <= INT32_MAX";
  if (io.lag < 0 || io.lag > DEXR_FIXED_LAG_MAX) return "lag must be in 0..4095";
  if (S > INT32_MAX / ((long long)io.lag + 1)) return "num_streams * (lag + 1) must be <= INT32_MAX";
  if (prm.preprocess != 0) return "raw landmarks are not smoothed: params.preprocess must be 0 (pre-process the keypoints first)";
  if (!io.last_qpos || !io.window_keypoints || !io.window_qpos || !io.window_len)
    return "last_qpos, window_keypoints, window_qpos and window_len are required";
  if (K > 0 && (!io.keypoints || !io.qpos_out)) return "keypoints and qpos_out are required";
  if (t.len_proj > 0 && !io.projected) return "the robot has DexPilot flags but projected is NULL";
  if (t.n_fixed > 0 && (!io.window_fixed_qpos || (K > 0 && !io.fixed_qpos)))
    return "the robot has fixed joints but window_fixed_qpos or fixed_qpos is NULL";
  if (!(io.smooth_weight < 0.f) && !(io.smooth_weight >= 0.f && io.smooth_weight <= 3.0e38f))
    return "smooth_weight must be finite (< 0: params.norm_delta)";
  if (S > 0 && (!io.workspace || io.workspace_bytes < fixed_lag_workspace_bytes(t, S, io.lag)))
    return "workspace smaller than dexr_fixed_lag_workspace_bytes(robot, num_streams, lag)";
  return nullptr;
}

// The extra argument checks of dexr_fixed_lag_step_accel (after fixed_lag_io_error): nullptr, or what is wrong.
inline const char* fixed_lag_accel_error(const dexr_table_t& t, const dexr_fixed_lag_t& io, const dexr_fixed_lag_accel_t& acc,
                                         long long S) {
  if (!(acc.accel_weight > 0.f && acc.accel_weight <= 3.0e38f))
    return "accel_weight must be finite and > 0 (c = 0 streams use dexr_fixed_lag_step)";
  if (S > 0 && (!acc.prev_qpos || !acc.has_prev)) return "prev_qpos and has_prev are required";
  if (S > 0 && io.workspace_bytes < fixed_lag_accel_workspace_bytes(t, S, io.lag))
    return "workspace smaller than dexr_fixed_lag_accel_workspace_bytes(robot, num_streams, lag)";
  return nullptr;
}

// Advances the committed DexPilot flags `flags` (nullptr: none) by one step of the hysteresis recurrence with the frame at
// `kp`: prepare_targets' flag update alone, so the flags are those the smoother's walk holds after that frame (it reads only
// the human vectors).  Lanes below len_proj own one flag each; the second-stage flags read the first stage's by shuffles.
template <int G>
__device__ __forceinline__ void fixed_lag_advance_flags(const Solver<G, 0>& sv, const Dims& dm, const dexr_params_t& prm,
                                                        const float* kp, uint8_t* flags, bool live) {
  if (flags == nullptr || dm.loss != DEXR_LOSS_DEXPILOT) return;  // (uniform)
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l, len_s1 = dm.len_s1, len_proj = dm.len_proj;
  float tx = 0.f, ty = 0.f, tz = 0.f;
  if (live && l < dm.n_res) {
    const int ht = st.res_ht[l], ho = st.res_ho[l];
    tx = kp[3 * ht]; ty = kp[3 * ht + 1]; tz = kp[3 * ht + 2];
    if (ho >= 0) { tx -= kp[3 * ho]; ty -= kp[3 * ho + 1]; tz -= kp[3 * ho + 2]; }
  }
  const float dist = sqrtf(fmaf(tx, tx, fmaf(ty, ty, tz * tz)));
  int flag = 0;
  if (l < len_s1) {
    flag = live ? flags[l] : 0;
    if (dist < prm.project_dist) flag = 1;
    if (dist > prm.escape_dist) flag = 0;
  }
  const int k2 = l - len_s1;
  const bool is_s2 = (l >= len_s1) && (l < len_proj);
  const int so = is_s2 ? st.s2_origin[k2] : 0, sk = is_s2 ? st.s2_task[k2] : 0;
  const int fo = gshfl_i<G>(flag, so), fk_ = gshfl_i<G>(flag, sk);
  if (is_s2) flag = (fo && fk_ && dist <= 0.03f) ? 1 : 0;
  if (live && l < len_proj) flags[l] = (uint8_t)flag;
  __syncwarp();
}

// The frame at window slot j of stream s: writes its qpos (var lanes) and scatter + mimic (joint lanes) to row `row` of
// qpos_out / robot_qpos_out, NaN when `emit` is false; robot_qpos as the smoother's output composes it.  Returns x.
template <int G>
__device__ __forceinline__ float fixed_lag_emit(Solver<G, 0>& sv, const dexr_fixed_lag_t& io, const Dims& dm, long long s,
                                                int j, bool emit, bool live, float* qpos_out, float* robot_qpos_out,
                                                long long row) {
  const int l = sv.l, W1 = io.lag + 1;
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const long long slot = s * W1 + j;
  const bool rd = live && emit;
  const float x = (rd && sv.var >= 0) ? io.window_qpos[slot * dm.n_var + sv.var] : 0.f;
  sv.qfix = (rd && fixedi >= 0) ? io.window_fixed_qpos[slot * dm.n_fixed + fixedi] : 0.f;
  const float q = sv.compose_q(x);
  const float nan = __int_as_float(0x7fc00000);
  if (live) {
    if (qpos_out && sv.var >= 0) qpos_out[row * dm.n_var + sv.var] = emit ? x : nan;
    if (robot_qpos_out && l < dm.dof) robot_qpos_out[row * dm.dof + l] = emit ? q : nan;
  }
  return x;
}

// Before a commit of an acceleration-penalised stream s: the anchor (raw) becomes prev_qpos and has_prev is set (each var
// lane moves its own entry; the caller's __syncwarp orders lane 0's has_prev for the next solve).
template <int G>
__device__ __forceinline__ void fixed_lag_commit_pre(const Solver<G, 0>& sv, const dexr_fixed_lag_t& io,
                                                     const dexr_fixed_lag_accel_t& acc, const Dims& dm, long long s,
                                                     bool owner) {
  if (owner && sv.var >= 0) acc.prev_qpos[s * dm.n_var + sv.var] = io.last_qpos[s * dm.n_var + sv.var];
  if (owner && sv.l == 0) acc.has_prev[s] = 1;
}

// One tick of dexr_fixed_lag_step: tick pos[1] of stream pos[0] (< S).  `pos` is the caller's loop state, read again after
// the window solve: no index of the driver stays in a register across the smoother, which uses every register the 16-lane
// kernel has (128); window_len is stored before the solve (the count includes the incoming frame from the append on) and
// read back after it for the same reason.  `owner`: this group runs the stream (the kernel gives a 16-lane warp's second
// group none: it walks the same ticks with every read and write off, so that the warp's shuffles stay converged; it reads
// window_len too).  `wstatus`: the status words after the smoother's part of the workspace.  Between a lane's global
// writes and another lane's reads, __syncwarp.  REC (dexr_fixed_lag_step_tape): after the solve, the window minimiser goes
// to tape_qpos [S,K,L+1,n_var] and the committed flags the solve started from to tape_projected [S,K,len_proj] (nullptr:
// none).  ACC (dexr_fixed_lag_step_accel): the window solve is smooth_packed_stream<G, true, true> with c =
// acc->accel_weight and the stream's pre-anchor; a commit first moves the old anchor to prev_qpos and sets has_prev.
template <int G, bool REC = false, bool ACC = false>
__device__ __forceinline__ void fixed_lag_tick(Solver<G, 0>& sv, const dexr_fixed_lag_t& io, const Dims& dm,
                                               const dexr_params_t& prm, int32_t* wstatus, int K,
                                               const volatile long long* pos, bool owner, float* tape_qpos = nullptr,
                                               uint8_t* tape_projected = nullptr,
                                               const dexr_fixed_lag_accel_t* acc = nullptr) {
  constexpr int KP = 3 * DEXR_NUM_KEYPOINTS;
  const int l = sv.l, n = dm.n_var, nf = dm.n_fixed, L = io.lag, W1 = L + 1;
  const bool isvar = sv.var >= 0;
  {  // 1. append the frame at slot h
    const long long s = pos[0], fin = s * K + pos[1];
    const int h0 = io.window_len[s];
    const int h = h0 < 0 ? 0 : (h0 > L ? L : h0);  // (a count outside 0..L reads as the nearest bound)
    const long long wh = s * W1 + h;
    const int fixedi = Solver<G, 0>::ST().fixed_index[l];
    __syncwarp();  // (every lane has read window_len)
    if (owner) {
      for (int e = l; e < KP; e += G) io.window_keypoints[wh * KP + e] = io.keypoints[fin * KP + e];
      if (fixedi >= 0) io.window_fixed_qpos[wh * nf + fixedi] = io.fixed_qpos[fin * nf + fixedi];
      if (isvar) io.window_qpos[wh * n + sv.var] = h > 0 ? io.window_qpos[(wh - 1) * n + sv.var] : io.last_qpos[s * n + sv.var];
      if (l == 0) io.window_len[s] = h + 1;
    }
    __syncwarp();
  }
  {  // 2. the window solve: the smoother on packed stream s of the window arrays, frames s (L+1) .. s (L+1) + h
    const long long s = pos[0];
    dexr_smooth_t sio{};
    sio.keypoints = io.window_keypoints;
    sio.fixed_qpos = io.window_fixed_qpos;
    sio.last_qpos = io.last_qpos;
    sio.projected = io.projected;
    sio.qpos_init = io.window_qpos;
    sio.qpos_out = io.window_qpos;
    sio.status_out = wstatus;
    sio.workspace = io.workspace;
    if constexpr (ACC) {
      sio.smooth_weight = acc->accel_weight;  // (w is in sv.prm.norm_delta)
      sio.cost_out = reinterpret_cast<float*>(const_cast<dexr_fixed_lag_accel_t*>(acc));  // (pre_anchor_state)
      smooth_packed_stream<G, true, true>(sv, sio, dm, prm, PackedStream{s, s * W1, io.window_len[s]}, owner,
                                          static_cast<float*>(io.workspace));
    } else {
      smooth_packed_stream(sv, sio, dm, prm, PackedStream{s, s * W1, io.window_len[s]}, owner, static_cast<float*>(io.workspace));
    }
  }
  if constexpr (REC) {  // (each var lane copies the entries it wrote itself)
    const long long s = pos[0], t = s * K + pos[1];
    const int m = static_cast<const volatile int32_t*>(io.window_len)[s];
    if (owner && isvar)
      for (int j = 0; j < m; ++j) tape_qpos[(t * W1 + j) * n + sv.var] = io.window_qpos[(s * W1 + j) * n + sv.var];
    if (owner && tape_projected && l < dm.len_proj) tape_projected[t * dm.len_proj + l] = io.projected[s * dm.len_proj + l];
  }
  // 3. emit slot 0 and commit it, or emit nothing
  const long long s = pos[0], fin = s * K + pos[1], w0 = s * W1;
  const bool full = static_cast<const volatile int32_t*>(io.window_len)[s] == W1;
  const float x = fixed_lag_emit(sv, io, dm, s, 0, full, owner, io.qpos_out, io.robot_qpos_out, fin);
  if (owner && l == 0 && io.status_out) io.status_out[fin] = full ? wstatus[w0] : DEXR_STATUS_PENDING;
  if (full) {
    if constexpr (ACC) fixed_lag_commit_pre(sv, io, *acc, dm, s, owner);
    if (owner && isvar) io.last_qpos[s * n + sv.var] = x;
    fixed_lag_advance_flags(sv, dm, prm, io.window_keypoints + w0 * KP,
                            dm.len_proj > 0 ? io.projected + s * dm.len_proj : nullptr, owner);
    const int fixedi = Solver<G, 0>::ST().fixed_index[l];
    if (owner) {  // shift the window down by one (each lane moves the entries it owns)
      for (int j = 0; j < L; ++j) {
        for (int e = l; e < KP; e += G) io.window_keypoints[(w0 + j) * KP + e] = io.window_keypoints[(w0 + j + 1) * KP + e];
        if (fixedi >= 0) io.window_fixed_qpos[(w0 + j) * nf + fixedi] = io.window_fixed_qpos[(w0 + j + 1) * nf + fixedi];
        if (isvar) io.window_qpos[(w0 + j) * n + sv.var] = io.window_qpos[(w0 + j + 1) * n + sv.var];
      }
      if (l == 0) io.window_len[s] = L;
    }
  }
  __syncwarp();
}

// The flush of stream s (< S) of dexr_fixed_lag_step: the held frames as the last solve left them, in order; the last becomes
// the anchor, the flags advance through them and the window empties.  `owner` as in fixed_lag_tick.  ACC: each commit moves
// the anchor to the pre-anchor first (fixed_lag_commit_pre), as a tick's does.
template <int G, bool ACC = false>
__device__ __forceinline__ void fixed_lag_flush(Solver<G, 0>& sv, const dexr_fixed_lag_t& io, const Dims& dm,
                                                const dexr_params_t& prm, long long s, bool owner,
                                                const dexr_fixed_lag_accel_t* acc = nullptr) {
  const int l = sv.l, L = io.lag, W1 = L + 1;
  const int h0 = io.window_len[s];
  const int h = h0 < 0 ? 0 : (h0 > L ? L : h0);
  uint8_t* const flags = dm.len_proj > 0 ? io.projected + s * dm.len_proj : nullptr;
  for (int j = 0; j < L; ++j) {
    const bool held = j < h;
    const float x = fixed_lag_emit(sv, io, dm, s, j, held, owner, io.flush_qpos_out, io.flush_robot_qpos_out, s * L + j);
    if (held) {
      if constexpr (ACC) fixed_lag_commit_pre(sv, io, *acc, dm, s, owner);
      if (owner && sv.var >= 0) io.last_qpos[s * dm.n_var + sv.var] = x;
      fixed_lag_advance_flags(sv, dm, prm, io.window_keypoints + (s * W1 + j) * (3 * DEXR_NUM_KEYPOINTS), flags, owner);
    }
  }
  __syncwarp();  // (every lane has read window_len)
  if (owner && l == 0) {
    io.flush_count_out[s] = h;
    io.window_len[s] = 0;
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// backpropagation through fixed-lag smoothing (dexr_fixed_lag_step_vjp, see dexr.h for the math): each differentiated tick's
// window is rebuilt in the workspace as a one-stream packed clip and smooth_vjp_packed_stream runs unchanged on it
// ------------------------------------------------------------------------------------------------
// The workspace of a call on S streams of lag L, W1 = L + 1 frames per stream: the rebuilt windows (frames s W1 .. s W1 +
// m - 1 of stream s) and their outputs, and the per-stream rows of the smoother's view.  Stream s is packed stream 2 s of
// that view (offsets[2s], offsets[2s+1] bound its window), so that every window's range is its own two words; the odd
// streams are never run.  Each array starts on a 16-byte boundary.
struct FixedLagVjpWs {
  int64_t* offsets;  // [2S]
  float* smooth;     // [S W1] SmoothWs<G>::kFloats each: the smoother VJP's Z_t, y_t, v_t
  float* kp;         // [S W1,21,3] the window's keypoints
  float* fixed;      // [S W1,n_fixed]
  float* qpos;       // [S W1,n_var] the point X^k
  float* gq;         // [S W1,n_var] the window's qpos cotangent
  float* grq;        // [S W1,dof] the window's robot_qpos cotangent
  float* gkp;        // [S W1,21,3] the window VJP's keypoint cotangents
  float* gfixed;     // [S W1,n_fixed]
  int32_t* status;   // [S W1]
  float* anchor;     // [2S,n_var] row 2s: A_k
  float* ganchor;    // [2S,n_var] row 2s: the window VJP's anchor cotangent
  float* abar;       // [S,n_var] the carried anchor cotangent
  uint8_t* flags;    // [2S,len_proj] row 2s: the flags W_k's solve started from
};

// The accelerated backward's workspace after FixedLagVjpWs's arrays (dexr_fixed_lag_step_accel_vjp): there `smooth` holds
// SmoothAccWs<G>::kFloats per frame, row 2s + 1 of `anchor` the pre-anchor P_k of stream s's window and row 2s + 1 of
// `ganchor` its cotangent, and `abar` is C1.
struct FixedLagPreWs {
  int32_t* has;  // [2S] entry 2s: H_k (the window VJP's io.workspace_bytes, pre_anchor_vjp_on)
  float* cbar2;  // [S,n_var] C2, the carried cotangent of X^{k-1}[0]
};

// Lays the workspace of S streams of lag L out from `base` (may be nullptr) into `w`; returns its size in bytes.  `pw`
// (non-null: dexr_fixed_lag_step_accel_vjp's layout): the accel smoother's frames and the FixedLagPreWs arrays after the rest.
inline size_t fixed_lag_vjp_layout(const dexr_table_t& t, long long S, long long lag, void* base, FixedLagVjpWs* w,
                                   FixedLagPreWs* pw = nullptr) {
  if (S <= 0 || lag < 0 || lag > DEXR_FIXED_LAG_MAX) return 0;
  const long long F = S * (lag + 1);
  const int floats = pw ? (eval_lanes(t) == 16 ? SmoothAccWs<16>::kFloats : SmoothAccWs<32>::kFloats)
                        : (eval_lanes(t) == 16 ? SmoothWs<16>::kFloats : SmoothWs<32>::kFloats);
  char* const b = static_cast<char*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = b ? b + off : nullptr;
    off += (bytes + 15) & ~(size_t)15;
    return static_cast<void*>(p);
  };
  FixedLagVjpWs r;
  r.offsets = static_cast<int64_t*>(take((size_t)(2 * S) * sizeof(int64_t)));
  r.smooth = static_cast<float*>(take((size_t)F * floats * sizeof(float)));
  r.kp = static_cast<float*>(take((size_t)F * 3 * DEXR_NUM_KEYPOINTS * sizeof(float)));
  r.fixed = static_cast<float*>(take((size_t)F * t.n_fixed * sizeof(float)));
  r.qpos = static_cast<float*>(take((size_t)F * t.n_var * sizeof(float)));
  r.gq = static_cast<float*>(take((size_t)F * t.n_var * sizeof(float)));
  r.grq = static_cast<float*>(take((size_t)F * t.dof * sizeof(float)));
  r.gkp = static_cast<float*>(take((size_t)F * 3 * DEXR_NUM_KEYPOINTS * sizeof(float)));
  r.gfixed = static_cast<float*>(take((size_t)F * t.n_fixed * sizeof(float)));
  r.status = static_cast<int32_t*>(take((size_t)F * sizeof(int32_t)));
  r.anchor = static_cast<float*>(take((size_t)(2 * S) * t.n_var * sizeof(float)));
  r.ganchor = static_cast<float*>(take((size_t)(2 * S) * t.n_var * sizeof(float)));
  r.abar = static_cast<float*>(take((size_t)S * t.n_var * sizeof(float)));
  r.flags = static_cast<uint8_t*>(take((size_t)(2 * S) * t.len_proj));
  if (pw) {
    pw->has = static_cast<int32_t*>(take((size_t)(2 * S) * sizeof(int32_t)));
    pw->cbar2 = static_cast<float*>(take((size_t)S * t.n_var * sizeof(float)));
  }
  if (w) *w = r;
  return off;
}

// dexr_fixed_lag_vjp_workspace_bytes.
inline size_t fixed_lag_vjp_workspace_bytes(const dexr_table_t& t, long long S, long long lag) {
  return fixed_lag_vjp_layout(t, S, lag, nullptr, nullptr);
}

// dexr_fixed_lag_accel_vjp_workspace_bytes.
inline size_t fixed_lag_accel_vjp_workspace_bytes(const dexr_table_t& t, long long S, long long lag) {
  FixedLagPreWs pw;
  return fixed_lag_vjp_layout(t, S, lag, nullptr, nullptr, &pw);
}

// The smoother VJP's view of a laid-out workspace: packed clips of the rebuilt windows.
inline dexr_smooth_vjp_t fixed_lag_vjp_window_io(const dexr_table_t& t, const FixedLagVjpWs& w) {
  dexr_smooth_vjp_t v{};
  v.keypoints = w.kp;
  v.fixed_qpos = t.n_fixed > 0 ? w.fixed : nullptr;
  v.last_qpos = w.anchor;
  v.projected = t.len_proj > 0 ? w.flags : nullptr;
  v.qpos = w.qpos;
  v.grad_qpos = w.gq;
  v.grad_robot_qpos = w.grq;
  v.smooth_weight = -1.f;  // (not read by the kernel: params.norm_delta holds w)
  v.workspace = w.smooth;
  v.grad_keypoints = w.gkp;
  v.grad_fixed_qpos = t.n_fixed > 0 ? w.gfixed : nullptr;
  v.grad_last_qpos = w.ganchor;
  v.status_out = w.status;
  return v;
}

// The accelerated window VJP's view (smooth_vjp_packed_stream<G, true, true>): c in smooth_weight, the H_k flags in
// workspace_bytes (pre_anchor_vjp_on).
inline dexr_smooth_vjp_t fixed_lag_accel_vjp_window_io(const dexr_table_t& t, const FixedLagVjpWs& w, const FixedLagPreWs& pw,
                                                       float accel_weight) {
  dexr_smooth_vjp_t v = fixed_lag_vjp_window_io(t, w);
  v.smooth_weight = accel_weight;
  v.workspace_bytes = reinterpret_cast<size_t>(pw.has);
  return v;
}

// The argument checks of dexr_fixed_lag_step_tape's tape: nullptr, or what is wrong.
inline const char* fixed_lag_tape_error(const dexr_table_t& t, const dexr_fixed_lag_tape_t* tape) {
  if (!tape || !tape->qpos) return "tape->qpos is required";
  if (t.len_proj > 0 && !tape->projected) return "DexPilot: the flag tape needs tape->projected";
  return nullptr;
}

// The argument checks of dexr_fixed_lag_step_vjp: nullptr, or what is wrong.  Host code shared by the library and the host
// emulation.
inline const char* fixed_lag_vjp_io_error(const dexr_table_t& t, const dexr_fixed_lag_vjp_t& io, const dexr_params_t& prm,
                                          long long S, long long K) {
  if (S < 0 || K < 0 || K > INT32_MAX) return "bad sizes: num_streams and num_ticks must be >= 0, num_ticks <= INT32_MAX";
  if (io.lag < 0 || io.lag > DEXR_FIXED_LAG_MAX) return "lag must be in 0..4095";
  if (S > INT32_MAX / (2 * ((long long)io.lag + 1))) return "num_streams * (lag + 1) must be <= INT32_MAX / 2";
  if (prm.preprocess != 0) return "raw landmarks are not differentiated: params.preprocess must be 0 (pre-process the keypoints first)";
  if (!io.last_qpos || !io.window_len) return "last_qpos and window_len (the state before the call) are required";
  if (K > 0 && (!io.keypoints || !io.window_keypoints || !io.tape.qpos || !io.grad_keypoints))
    return "keypoints, window_keypoints, tape.qpos and grad_keypoints are required";
  if (K > 0 && t.len_proj > 0 && !io.tape.projected) return "DexPilot: tape.projected is required";
  if (K > 0 && t.n_fixed > 0 && (!io.fixed_qpos || !io.window_fixed_qpos))
    return "the robot has fixed joints but fixed_qpos or window_fixed_qpos is NULL";
  if (!(io.smooth_weight < 0.f) && !(io.smooth_weight >= 0.f && io.smooth_weight <= 3.0e38f))
    return "smooth_weight must be finite (< 0: params.norm_delta)";
  if (S > 0 && (!io.workspace || io.workspace_bytes < fixed_lag_vjp_workspace_bytes(t, S, io.lag)))
    return "workspace smaller than dexr_fixed_lag_vjp_workspace_bytes(robot, num_streams, lag)";
  return nullptr;
}

// The extra argument checks of dexr_fixed_lag_step_accel_vjp (after fixed_lag_vjp_io_error): nullptr, or what is wrong.
inline const char* fixed_lag_accel_vjp_error(const dexr_table_t& t, const dexr_fixed_lag_vjp_t& io,
                                             const dexr_fixed_lag_accel_vjp_t& acc, long long S) {
  if (!(acc.accel_weight > 0.f && acc.accel_weight <= 3.0e38f))
    return "accel_weight must be finite and > 0 (c = 0 streams use dexr_fixed_lag_step_vjp)";
  if (S > 0 && (!acc.prev_qpos || !acc.has_prev)) return "prev_qpos and has_prev (the state before the call) are required";
  if (S > 0 && io.workspace_bytes < fixed_lag_accel_vjp_workspace_bytes(t, S, io.lag))
    return "workspace smaller than dexr_fixed_lag_accel_vjp_workspace_bytes(robot, num_streams, lag)";
  return nullptr;
}

// Where a stream's call ends (group-uniform): h0 the held frames at the start, hend those held after the ticks (before a
// flush), cend the frames committed by then (final slot i holds input frame cend + i), elast whether the last tick emitted
// and `route` where grad_last_qpos_out goes: 0 the incoming anchor, 1 slot 0 of the last window, 2 its last held slot.
struct FixedLagEnd {
  int h0, hend, cend, elast, route;
};
__device__ __forceinline__ FixedLagEnd fixed_lag_end(int h0_raw, int L, int K, bool flushed) {
  FixedLagEnd e;
  e.h0 = h0_raw < 0 ? 0 : (h0_raw > L ? L : h0_raw);
  const int mlast = K > 0 ? (e.h0 + K < L + 1 ? e.h0 + K : L + 1) : e.h0;
  e.elast = (K > 0 && mlast == L + 1) ? 1 : 0;
  e.hend = mlast - e.elast;
  e.cend = e.h0 + K - L > 0 ? e.h0 + K - L : 0;
  e.route = (flushed && e.hend > 0) ? 2 : (e.elast ? 1 : 0);
  return e;
}

// Where grad_prev_qpos_out goes (dexr_fixed_lag_step_accel_vjp): the final prev_qpos is commit i = N - 2 of the call's N =
// cend + (flushed ? hend : 0) commits, the incoming pre-anchor and anchor counting as commits -2 and -1.  0: the incoming
// pre-anchor (grad_prev_qpos), 1: the incoming anchor (grad_last_qpos), 2: X^{K-2}[0] (C2 at the start), 3: X^{K-1}[0]
// (slot 0 of the last window), 4: the flushed slot hend - 2.
__device__ __forceinline__ int fixed_lag_pre_route(const FixedLagEnd& e, bool flushed) {
  const int i = e.cend + (flushed ? e.hend : 0) - 2;
  return i == -2 ? 0 : (i == -1 ? 1 : (i >= e.cend ? 4 : (i == e.cend - 1 ? 3 : 2)));
}

// smooth_vjp_packed_stream's cotangent of a var lane: M^T r (r: this lane's joint's robot_qpos cotangent, the mimic
// followers folded into their source) + gq, in its order of operations, so that a cotangent folded here and one folded by
// the window VJP give the same bits.
template <int G>
__device__ __forceinline__ float fixed_lag_fold(const Solver<G, 0>& sv, const Dims& dm, float r, float gq) {
  const SharedTable& st = Solver<G, 0>::ST();
  const int l = sv.l;
  const bool isvar = sv.var >= 0;
  float gb = r;
  if (dm.has_mimic) {
    const int gcount = st.group_count[l];
    float gx_ = 0.f;
#pragma unroll
    for (int k = 0; k < DEXR_MAX_GROUP; ++k) {
      const bool v = isvar && k < gcount;
      const float gv = gshfl<G>(r, v ? st.group_lane[l][k] : l);
      if (v) gx_ = fmaf(st.group_mult[l][k], gv, gx_);
    }
    gb = gx_;
  }
  gb += gq;
  return isvar ? gb : 0.f;
}

// The start of stream s (< S) of dexr_fixed_lag_step_vjp: every output row of the stream written once (zeros, PENDING), the
// final state's keypoint and fixed-joint cotangents onto the input frames their held slots hold (the flushed rows' fixed-joint
// share too: those frames' sums start with it, so a chunked run gives the same bits; unlike the window VJP's direct term
// it is kept on a NOT_PD window or a missing frame, see dexr.h), the anchor's own cotangent when it routes there, the carried abar zeroed.
// With K = 0 the flush rows are the incoming held slots of window_qpos.  `owner` as in fixed_lag_tick.  ACC
// (dexr_fixed_lag_step_accel_vjp, with `acc` and the workspace's `pw`): grad_prev_qpos_out goes where fixed_lag_pre_route
// sends it (grad_last_qpos or grad_prev_qpos written with it, C2 started with it, or a flushed slot's sum), C2 zeroed
// otherwise; the last window's slot 0 takes it in fixed_lag_vjp_rebuild.
template <int G, bool ACC = false>
__device__ __forceinline__ void fixed_lag_vjp_begin(const Solver<G, 0>& sv, const dexr_fixed_lag_vjp_t& io,
                                                    const FixedLagVjpWs& ws, const Dims& dm, long long s, int K,
                                                    bool owner, const dexr_fixed_lag_accel_vjp_t* acc = nullptr,
                                                    const FixedLagPreWs* pw = nullptr) {
  constexpr int KP = 3 * DEXR_NUM_KEYPOINTS;
  const int l = sv.l, n = dm.n_var, nf = dm.n_fixed, dof = dm.dof, L = io.lag, W1 = L + 1;
  const bool isvar = sv.var >= 0;
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const FixedLagEnd e = fixed_lag_end(io.window_len[s], L, K, io.flushed != 0);
  if (owner) {
    for (int k = 0; k < K; ++k) {
      for (int c = l; c < KP; c += G) io.grad_keypoints[(s * K + k) * KP + c] = 0.f;
      if (fixedi >= 0 && io.grad_fixed_qpos) io.grad_fixed_qpos[(s * K + k) * nf + fixedi] = 0.f;
      if (l == 0 && io.status_out) io.status_out[s * K + k] = DEXR_STATUS_PENDING;
    }
    for (int j = 0; j < W1; ++j) {
      if (io.grad_window_keypoints)
        for (int c = l; c < KP; c += G) io.grad_window_keypoints[(s * W1 + j) * KP + c] = 0.f;
      if (fixedi >= 0 && io.grad_window_fixed_qpos) io.grad_window_fixed_qpos[(s * W1 + j) * nf + fixedi] = 0.f;
      if (isvar && io.grad_window_qpos) io.grad_window_qpos[(s * W1 + j) * n + sv.var] = 0.f;
    }
    if (isvar) {
      if (io.grad_last_qpos)
        io.grad_last_qpos[s * n + sv.var] = (e.route == 0 && io.grad_last_qpos_out) ? io.grad_last_qpos_out[s * n + sv.var] : 0.f;
      ws.abar[s * n + sv.var] = 0.f;
      if constexpr (ACC) {  // (route 1 is never the anchor's route 0: at most one of the two writes grad_last_qpos)
        const int pr = fixed_lag_pre_route(e, io.flushed != 0);
        const float gp = acc->grad_prev_qpos_out ? acc->grad_prev_qpos_out[s * n + sv.var] : 0.f;
        if (pr == 1 && io.grad_last_qpos) io.grad_last_qpos[s * n + sv.var] = gp;
        if (acc->grad_prev_qpos) acc->grad_prev_qpos[s * n + sv.var] = pr == 0 ? gp : 0.f;
        pw->cbar2[s * n + sv.var] = pr == 2 ? gp : 0.f;
      }
    }
    // the final state's held slots: slot i holds input frame g = cend + i (held at the start when g < h0)
    for (int i = 0; i < e.hend; ++i) {
      const int g = e.cend + i;
      const bool held = g < e.h0;
      if (io.grad_window_keypoints_out) {
        float* const d = held ? io.grad_window_keypoints : io.grad_keypoints;
        const long long row = held ? s * W1 + g : s * K + (g - e.h0);
        if (d)
          for (int c = l; c < KP; c += G) d[row * KP + c] = io.grad_window_keypoints_out[(s * W1 + i) * KP + c];
      }
      if (fixedi >= 0) {
        float* const d = held ? io.grad_window_fixed_qpos : io.grad_fixed_qpos;
        const long long row = held ? s * W1 + g : s * K + (g - e.h0);
        float v = io.grad_window_fixed_qpos_out ? io.grad_window_fixed_qpos_out[(s * W1 + i) * nf + fixedi] : 0.f;
        if (io.flushed && io.grad_flush_robot_qpos) v += io.grad_flush_robot_qpos[(s * L + i) * dof + l];
        if (d) d[row * nf + fixedi] = v;
      }
    }
  }
  __syncwarp();
  if (K == 0) {  // (uniform) the held slots of window_qpos are the flushed rows and the final window_qpos
    for (int j = 0; j < e.h0; ++j) {
      const float r = (owner && l < dof && io.flushed && io.grad_flush_robot_qpos && fixedi < 0)
                          ? io.grad_flush_robot_qpos[(s * L + j) * dof + l] : 0.f;
      float q = 0.f;
      if (owner && isvar) {
        q = io.grad_window_qpos_out ? io.grad_window_qpos_out[(s * W1 + j) * n + sv.var] : 0.f;
        q += (io.flushed && io.grad_flush_qpos) ? io.grad_flush_qpos[(s * L + j) * n + sv.var] : 0.f;
        if (e.route == 2 && j == e.h0 - 1 && io.grad_last_qpos_out) q += io.grad_last_qpos_out[s * n + sv.var];
        if constexpr (ACC)
          if (fixed_lag_pre_route(e, io.flushed != 0) == 4 && j == e.h0 - 2 && acc->grad_prev_qpos_out)
            q += acc->grad_prev_qpos_out[s * n + sv.var];
      }
      const float gb = fixed_lag_fold(sv, dm, r, q);
      if (owner && isvar && io.grad_window_qpos) io.grad_window_qpos[(s * W1 + j) * n + sv.var] = gb;
    }
  }
  __syncwarp();
}

// Rebuilds the window of tick pos[1] of stream pos[0] of dexr_fixed_lag_step_vjp in the workspace (frames, fixed joints,
// point, anchor, flags and the slot cotangents, see dexr.h) when the tick is differentiated -- it emits or is the last --
// and returns whether it is (group-uniform).  `owner` as in fixed_lag_tick.  ACC: also the pre-anchor P_k (row 2s + 1 of
// ws.anchor: prev_qpos when c_k = 0, last_qpos when c_k = 1, X^{k-2}[0] otherwise) and H_k (has_prev when c_k = 0, else 1),
// and grad_prev_qpos_out on the slot fixed_lag_pre_route gives it.
template <int G, bool ACC = false>
__device__ __forceinline__ bool fixed_lag_vjp_rebuild(const Solver<G, 0>& sv, const dexr_fixed_lag_vjp_t& io,
                                                      const FixedLagVjpWs& ws, const Dims& dm, int K,
                                                      const volatile long long* pos, bool owner,
                                                      const dexr_fixed_lag_accel_vjp_t* acc = nullptr,
                                                      const FixedLagPreWs* pw = nullptr) {
  constexpr int KP = 3 * DEXR_NUM_KEYPOINTS;
  const int l = sv.l, n = dm.n_var, nf = dm.n_fixed, dof = dm.dof, L = io.lag, W1 = L + 1;
  const long long s = pos[0];
  const int k = (int)pos[1];
  const FixedLagEnd e = fixed_lag_end(io.window_len[s], L, K, io.flushed != 0);
  const int m = e.h0 + k + 1 < W1 ? e.h0 + k + 1 : W1, c0 = e.h0 + k - L > 0 ? e.h0 + k - L : 0;
  const bool emit = m == W1, last = k == K - 1;
  if (!emit && !last) {
    __syncwarp();  // (every lane has read the loop state and window_len before lane 0 advances the loop)
    return false;
  }
  const bool isvar = sv.var >= 0;
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const long long t = s * K + k, w0 = s * W1;
  if (owner) {
    for (int j = 0; j < m; ++j) {
      const int g = c0 + j;
      const bool held = g < e.h0;
      const long long src = held ? s * W1 + g : s * K + (g - e.h0);
      const float* const kp = held ? io.window_keypoints : io.keypoints;
      for (int c = l; c < KP; c += G) ws.kp[(w0 + j) * KP + c] = kp[src * KP + c];
      if (fixedi >= 0) ws.fixed[(w0 + j) * nf + fixedi] = (held ? io.window_fixed_qpos : io.fixed_qpos)[src * nf + fixedi];
      // the slot's cotangents: slot 0 of an emitting tick its emitted row (+ abar, or grad_last_qpos_out on the last tick);
      // on the last tick the slots still held after it (final slot i = j - elast) the final state's and the flush's
      const int i = j - e.elast;
      const bool row = emit && j == 0, tail = last && i >= 0;
      if (isvar) {
        ws.qpos[(w0 + j) * n + sv.var] = io.tape.qpos[(t * W1 + j) * n + sv.var];
        float q = 0.f;
        if (row) {
          q = io.grad_qpos ? io.grad_qpos[t * n + sv.var] : 0.f;
          if (!last) q += ws.abar[s * n + sv.var];
          else if (e.route == 1 && io.grad_last_qpos_out) q += io.grad_last_qpos_out[s * n + sv.var];
          if constexpr (ACC)  // (route 3: the anchor's route is 2, so nothing else was added)
            if (last && fixed_lag_pre_route(e, io.flushed != 0) == 3 && acc->grad_prev_qpos_out)
              q += acc->grad_prev_qpos_out[s * n + sv.var];
        } else if (tail) {
          q = io.grad_window_qpos_out ? io.grad_window_qpos_out[(w0 + i) * n + sv.var] : 0.f;
          q += (io.flushed && io.grad_flush_qpos) ? io.grad_flush_qpos[(s * L + i) * n + sv.var] : 0.f;
          if (e.route == 2 && i == e.hend - 1 && io.grad_last_qpos_out) q += io.grad_last_qpos_out[s * n + sv.var];
          if constexpr (ACC)
            if (fixed_lag_pre_route(e, io.flushed != 0) == 4 && i == e.hend - 2 && acc->grad_prev_qpos_out)
              q += acc->grad_prev_qpos_out[s * n + sv.var];
        }
        ws.gq[(w0 + j) * n + sv.var] = q;
      }
      if (l < dof) {  // (a flushed row's fixed-joint share went to the frame's sum in fixed_lag_vjp_begin)
        float r = 0.f;
        if (row) r = io.grad_robot_qpos ? io.grad_robot_qpos[t * dof + l] : 0.f;
        else if (tail && fixedi < 0 && io.flushed && io.grad_flush_robot_qpos) r = io.grad_flush_robot_qpos[(s * L + i) * dof + l];
        ws.grq[(w0 + j) * dof + l] = r;
      }
    }
    if (isvar) ws.anchor[2 * s * n + sv.var] = c0 == 0 ? io.last_qpos[s * n + sv.var] : io.tape.qpos[((t - 1) * W1) * n + sv.var];
    if constexpr (ACC) {
      if (isvar)
        ws.anchor[(2 * s + 1) * n + sv.var] = c0 == 0 ? acc->prev_qpos[s * n + sv.var]
                                              : (c0 == 1 ? io.last_qpos[s * n + sv.var] : io.tape.qpos[((t - 2) * W1) * n + sv.var]);
      if (l == 0) pw->has[2 * s] = c0 == 0 ? (acc->has_prev[s] != 0 ? 1 : 0) : 1;
    }
    if (l < dm.len_proj) ws.flags[2 * s * dm.len_proj + l] = io.tape.projected[t * dm.len_proj + l];
    if (l == 0) {
      ws.offsets[2 * s] = w0;
      ws.offsets[2 * s + 1] = w0 + m;
    }
  }
  __syncwarp();
  return true;
}

// After the window VJP of tick pos[1] of stream pos[0]: its frames' cotangents added to the input frames they came from, its
// anchor cotangent carried to the previous tick's slot 0 (c_k >= 1) or added to grad_last_qpos (c_k = 0), the emitted
// frame's status.  ACC, with ga the window's anchor cotangent and gp its pre-anchor's: c_k >= 1: C1 = C2 + ga; c_k = 0:
// grad_last_qpos += ga; then c_k >= 2: C2 = gp; c_k = 1: grad_last_qpos += gp; c_k = 0: grad_prev_qpos += gp.
template <int G, bool ACC = false>
__device__ __forceinline__ void fixed_lag_vjp_scatter(const Solver<G, 0>& sv, const dexr_fixed_lag_vjp_t& io,
                                                      const FixedLagVjpWs& ws, const Dims& dm, int K,
                                                      const volatile long long* pos, bool owner,
                                                      const dexr_fixed_lag_accel_vjp_t* acc = nullptr,
                                                      const FixedLagPreWs* pw = nullptr) {
  constexpr int KP = 3 * DEXR_NUM_KEYPOINTS;
  const int l = sv.l, n = dm.n_var, nf = dm.n_fixed, L = io.lag, W1 = L + 1;
  const long long s = pos[0];
  const int k = (int)pos[1];
  const int h0r = io.window_len[s];
  const int h0 = h0r < 0 ? 0 : (h0r > L ? L : h0r);
  const int m = h0 + k + 1 < W1 ? h0 + k + 1 : W1, c0 = h0 + k - L > 0 ? h0 + k - L : 0;
  const int fixedi = Solver<G, 0>::ST().fixed_index[l];
  const long long w0 = s * W1;
  if (owner) {
    for (int j = 0; j < m; ++j) {
      const int g = c0 + j;
      const bool held = g < h0;
      const long long row = held ? s * W1 + g : s * K + (g - h0);
      float* const d = held ? io.grad_window_keypoints : io.grad_keypoints;
      if (d)
        for (int c = l; c < KP; c += G) d[row * KP + c] += ws.gkp[(w0 + j) * KP + c];
      float* const df = held ? io.grad_window_fixed_qpos : io.grad_fixed_qpos;
      if (fixedi >= 0 && df) df[row * nf + fixedi] += ws.gfixed[(w0 + j) * nf + fixedi];
    }
    if constexpr (ACC) {
      if (sv.var >= 0) {
        const float ab = ws.ganchor[2 * s * n + sv.var], gp = ws.ganchor[(2 * s + 1) * n + sv.var];
        float* const c2 = pw->cbar2 + s * n + sv.var;
        if (c0 > 0) ws.abar[s * n + sv.var] = *c2 + ab;
        else if (io.grad_last_qpos) io.grad_last_qpos[s * n + sv.var] += ab;
        if (c0 > 1) *c2 = gp;
        else if (c0 == 1) {
          if (io.grad_last_qpos) io.grad_last_qpos[s * n + sv.var] += gp;
        } else if (acc->grad_prev_qpos) {
          acc->grad_prev_qpos[s * n + sv.var] += gp;
        }
      }
    } else if (sv.var >= 0) {
      const float ab = ws.ganchor[2 * s * n + sv.var];
      if (c0 > 0) ws.abar[s * n + sv.var] = ab;
      else if (io.grad_last_qpos) io.grad_last_qpos[s * n + sv.var] += ab;
    }
    if (l == 0 && io.status_out && m == W1) io.status_out[s * K + k] = ws.status[w0];
  }
  __syncwarp();
}

}  // namespace dexr
