// dexr.cu -- kernels' entry points and the C ABI of libdexr.so (see include/dexr.h).
//
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include "dexr_kernels.cuh"

namespace dexr {

// ------------------------------------------------------------------------------------------------
// kernel arguments
// ------------------------------------------------------------------------------------------------
struct FrameArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_frames_t io;
  long long B;
  int T;          // frames per tile (multiple of 4)
  int ntiles;
  int use_bulk;   // inputs 16-byte aligned -> cp.async.bulk for full tiles
  int in_row;     // floats per frame of the kp/ref input (63 or 3m)
  Dims dm;
  int off_in, off_last, off_fixed, stage_bytes;  // ring stage layout (bytes)
  int ring_off, bar_off, scratch_off;            // dynamic smem layout (bytes)
};

struct SeqArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_sequences_t io;
  long long S;
  int steps;
  Dims dm;
  int scratch_off;
  int spw;  // streams per warp: 32 / G when streams are plentiful; 1 when they are scarce (a stream is latency bound, and two
            // streams sharing a warp both pay the larger of their two iteration counts on every frame)
  int duo;  // spw == 1 with a 16-lane solver: the second half-warp works on the SAME stream (Solver::duo) instead of idling
};

// ------------------------------------------------------------------------------------------------
// independent frames: producer warp (TMA ring) + NCW consumer warps
// ------------------------------------------------------------------------------------------------
// One robot group, executed by one CTA: the tiles `first_tile, first_tile + gridDim.x, ...` of the group's batch.  Both the
// single-robot kernel and the mixed-robot kernel (several groups back to back inside one launch) run this body; it starts
// and ends with a CTA-wide barrier, so it can be called repeatedly with different tables / template parameters.
template <int G, int BW, int NCW>
__device__ __forceinline__ void frames_group(const FrameArgs& a, int first_tile) {
  unsigned char* const smem = dsmem;
  SharedTable* st = reinterpret_cast<SharedTable*>(smem);
  unsigned char* ring = smem + a.ring_off;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + a.bar_off);
  uint64_t* empty = full + 2;
  int* next = reinterpret_cast<int*>(empty + 2);

  __syncthreads();  // (mixed launches: every warp is done with the previous group's table, ring and barriers)
  load_shared_table(*st, a.table, pass_slot_width<BW>());
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_init(&empty[0], NCW);
    mbar_init(&empty[1], NCW);
    next[0] = 0;
    next[1] = 0;
    mbar_fence_init();
  }
  __syncthreads();

  // warp-uniform by construction: tells the compiler that the role split below never splits a warp
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const bool by_kp = a.io.keypoints != nullptr;
  const float* g_in = by_kp ? a.io.keypoints : a.io.ref_value;

  if (warp == NCW) {
    // ===================== producer: stage tiles HBM -> shared memory =====================
    int it = 0;
    for (int tile = first_tile; tile < a.ntiles; tile += gridDim.x, ++it) {
      const int stage = it & 1;
      if (it >= 2) mbar_wait(&empty[stage], ((it >> 1) - 1) & 1);
      const long long f0 = (long long)tile * a.T;
      const int count = (int)min((long long)a.T, a.B - f0);
      unsigned char* sb = ring + stage * a.stage_bytes;
      float* s_in = reinterpret_cast<float*>(sb + a.off_in);
      float* s_last = reinterpret_cast<float*>(sb + a.off_last);
      float* s_fixed = reinterpret_cast<float*>(sb + a.off_fixed);
      const float* gi = g_in + f0 * a.in_row;
      const float* gl = a.io.last_qpos + f0 * a.dm.n_var;
      const float* gf = a.dm.n_fixed > 0 ? a.io.fixed_qpos + f0 * a.dm.n_fixed : nullptr;
      if (lane == 0) next[stage] = 0;
      if (a.use_bulk && (count & 3) == 0) {
        if (lane == 0) {
          const uint32_t b_in = (uint32_t)count * a.in_row * 4u;
          const uint32_t b_last = (uint32_t)count * a.dm.n_var * 4u;
          const uint32_t b_fixed = (uint32_t)count * a.dm.n_fixed * 4u;
          mbar_arrive_expect_tx(&full[stage], b_in + b_last + b_fixed);
          bulk_g2s(s_in, gi, b_in, &full[stage]);
          bulk_g2s(s_last, gl, b_last, &full[stage]);
          if (b_fixed) bulk_g2s(s_fixed, gf, b_fixed, &full[stage]);
        }
      } else {
        for (int i = lane; i < count * a.in_row; i += 32) s_in[i] = gi[i];
        for (int i = lane; i < count * a.dm.n_var; i += 32) s_last[i] = gl[i];
        for (int i = lane; i < count * a.dm.n_fixed; i += 32) s_fixed[i] = gf[i];
        __threadfence_block();  // every lane's stores are visible CTA-wide before lane 0 publishes the stage
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[stage]);
      }
      __syncwarp();
    }
  } else {
    // ===================== consumers: one frame per group of G lanes =========================
    constexpr int GPW = 32 / G;
    const int gid = warp * GPW + (lane / G);
    Solver<G, BW> sv;
    sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * Scratch<G>::kFloats * 4), a.prm, lane);

    int it = 0;
    for (int tile = first_tile; tile < a.ntiles; tile += gridDim.x, ++it) {
      const int stage = it & 1;
      mbar_wait(&full[stage], (it >> 1) & 1);
      const long long f0 = (long long)tile * a.T;
      const int count = (int)min((long long)a.T, a.B - f0);
      const unsigned char* sb = ring + stage * a.stage_bytes;
      const float* s_in = reinterpret_cast<const float*>(sb + a.off_in);
      const float* s_last = reinterpret_cast<const float*>(sb + a.off_last);
      const float* s_fixed = reinterpret_cast<const float*>(sb + a.off_fixed);
      while (true) {
        int base = 0;
        if (lane == 0) base = atomicAdd(&next[stage], GPW);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= count) break;
        const int idx = base + (lane / G);
        const bool active = idx < count;
        const int ci = active ? idx : base;
        const long long f = f0 + ci;
        FrameInputs in;
        in.kp = by_kp ? s_in + ci * a.in_row : nullptr;
        in.ref = by_kp ? nullptr : s_in + ci * a.in_row;
        in.last = s_last + ci * a.dm.n_var;
        in.fixed = s_fixed + ci * a.dm.n_fixed;
        in.projected = a.io.projected ? a.io.projected + f * a.dm.len_proj : nullptr;
        solve_frame(sv, in, a.io, a.dm, f, active);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
    }
  }
}

template <int G, int BW, int NCW>
__global__ void __launch_bounds__((NCW + 1) * 32, 1) dexr_frames_kernel(const FrameArgs a) {
  frames_group<G, BW, NCW>(a, blockIdx.x);
}

// ------------------------------------------------------------------------------------------------
// mixed robots: ONE persistent launch over a list of (robot table, frame batch) groups (the reference builds one optimizer
// per robot, retargeting_config.py:167-257, and would run them one after the other).  A CTA walks the groups in order; per
// group it reloads the 8 KB table into shared memory and re-arms the input ring (two CTA barriers), picks the solver
// instantiation the table asks for (16 / 32 lanes, block / dense / arrow Hessian) and takes every gridDim-th tile.  The
// round-robin over CTAs continues ACROSS groups (`rot`), so the CTAs that got one tile fewer in one group are first in line
// in the next.  There is no grid-wide barrier: a CTA that finishes a group early starts the next one, and the only tail
// of the launch is the last group's.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxGroups = DEXR_MAX_GROUPS;
struct MultiArgs {
  int n_groups;
  int kind[kMaxGroups];  // SolverKind
  FrameArgs g[kMaxGroups];
};

// A/B switch DEXR_EXP_MULTI_CALLS: a real call per solver instantiation (own register allocation per body, but the group's
// arguments then come through a pointer instead of the constant bank) instead of four inlined bodies in one allocation.
template <int G, int BW, int NCW>
#ifdef DEXR_EXP_MULTI_CALLS
__device__ __noinline__
#else
__device__ __forceinline__
#endif
void frames_group_call(const FrameArgs& a, int first_tile) {
  frames_group<G, BW, NCW>(a, first_tile);
}

template <int NCW>
__global__ void __launch_bounds__((NCW + 1) * 32, 1) dexr_frames_multi_kernel(const __grid_constant__ MultiArgs m) {
  int rot = 0;  // tiles handed out so far, modulo the grid: where the round-robin continues
  for (int gi = 0; gi < m.n_groups; ++gi) {
    const FrameArgs& a = m.g[gi];
    const int first = (int)((blockIdx.x + gridDim.x - rot) % gridDim.x);
    switch (m.kind[gi]) {
      case kBlock16: frames_group_call<16, 4, NCW>(a, first); break;
      case kDense16: frames_group_call<16, 0, NCW>(a, first); break;
      case kArrow32: frames_group_call<32, -1, NCW>(a, first); break;
      default: frames_group_call<32, 0, NCW>(a, first); break;
    }
    rot = (rot + a.ntiles) % gridDim.x;
  }
}

// ------------------------------------------------------------------------------------------------
// sequences: one group owns one stream and walks its T frames (seq_retarget.py:112-134)
// ------------------------------------------------------------------------------------------------
template <int G, int BW, int NW>
__global__ void __launch_bounds__(NW * 32, 1) dexr_sequences_kernel(const SeqArgs a) {
  unsigned char* const smem = dsmem;
  SharedTable* st = reinterpret_cast<SharedTable*>(smem);
  load_shared_table(*st, a.table, pass_slot_width<BW>());
  __syncthreads();

  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + (lane / G);               // scratch slot of this group of lanes
  const int slots_per_cta = NW * a.spw;
  const uint32_t scratch_off = (uint32_t)(a.scratch_off + gid * Scratch<G>::kStreamFloats * 4);
  float* kpbuf = reinterpret_cast<float*>(smem + scratch_off) + Scratch<G>::kFloats;  // 63 floats: current keypoints
  const int slot = a.spw == GPW ? gid : warp;            // which of the CTA's stream slots this group serves
  const bool first = (lane / G) == 0;
  const bool owner = a.spw == GPW || first;              // the group that reads and writes the stream's state
  const bool works = owner || a.duo;                     // (scarce streams, 16 lanes: the second half-warp helps the first)
  Solver<G, BW> sv;
  sv.init(a.table, a.dm, scratch_off, a.prm, lane);
  if (G == 16 && a.duo) sv.duo = lane / G;
  const bool use_filter = a.prm.lp_alpha >= 0.f && a.prm.lp_alpha <= 1.f;

  // Streams are dealt round-robin over CTAs (stream = blockIdx + gridDim * slot): with few streams every SM gets
  // one or two warps instead of a few SMs getting eight -- the path is latency bound per stream.
  for (long long base = 0; base < a.S; base += (long long)gridDim.x * slots_per_cta) {
    const long long s = base + (long long)slot * gridDim.x + blockIdx.x;
    solve_stream(sv, a.io, a.dm, a.prm, a.S, a.steps, s, works && s < a.S, owner && s < a.S, kpbuf, use_filter);
  }
}

// ------------------------------------------------------------------------------------------------
// keypoint pre-processing (single_hand_detector.py:100-103, 130-158): one thread per frame for the 3x3 frame,
// tile staged through shared memory so that global loads / stores are coalesced 16-byte accesses
// ------------------------------------------------------------------------------------------------
constexpr int kPreTile = 128;  // frames per CTA tile; 128 * 252 B = 32256 B, a multiple of 16

__global__ void __launch_bounds__(kPreTile) dexr_preprocess_kernel(const float* __restrict__ raw, float* __restrict__ out,
                                                                    float* __restrict__ rot_out, int left, long long B) {
  __shared__ __align__(16) float tile[kPreTile * 63];
  const int tid = threadIdx.x;
  for (long long f0 = (long long)blockIdx.x * kPreTile; f0 < B; f0 += (long long)gridDim.x * kPreTile) {
    const int count = (int)min((long long)kPreTile, B - f0);
    const int nfl = count * 63;
    const float* src = raw + f0 * 63;
    if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
      const float4* s4 = reinterpret_cast<const float4*>(src);
      float4* t4 = reinterpret_cast<float4*>(tile);
      for (int i = tid; i < nfl / 4; i += kPreTile) t4[i] = s4[i];
      for (int i = (nfl / 4) * 4 + tid; i < nfl; i += kPreTile) tile[i] = src[i];
    } else {
      for (int i = tid; i < nfl; i += kPreTile) tile[i] = src[i];
    }
    __syncthreads();
    if (tid < count) {
      float* k = tile + tid * 63;  // stride 63 floats: odd -> conflict-free per-thread rows
      const float wx = k[0], wy = k[1], wz = k[2];
      // landmarks 5 (index base) and 9 (middle base) relative to the wrist
      const float ax = k[15] - wx, ay = k[16] - wy, az = k[17] - wz;
      const float bx = k[27] - wx, by = k[28] - wy, bz = k[29] - wz;
      // plane normal through {wrist, index base, middle base}; the SVD of the reference gives +-this vector
      float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
      const float nn = rsqrtf(nx * nx + ny * ny + nz * nz);
      nx *= nn; ny *= nn; nz *= nn;
      // x axis: wrist - middle base, orthogonalised against the normal
      float xx = -bx, xy = -by, xz = -bz;
      const float dn = xx * nx + xy * ny + xz * nz;
      xx -= dn * nx; xy -= dn * ny; xz -= dn * nz;
      const float xn = rsqrtf(xx * xx + xy * xy + xz * xz);
      xx *= xn; xy *= xn; xz *= xn;
      float zx = xy * nz - xz * ny, zy = xz * nx - xx * nz, zz = xx * ny - xy * nx;
      // z should point like (index base - middle base)
      if (zx * (ax - bx) + zy * (ay - by) + zz * (az - bz) < 0.f) { nx = -nx; ny = -ny; nz = -nz; zx = -zx; zy = -zy; zz = -zz; }
      // frame = [x | normal | z] (columns); joint_pos = (kp - wrist) @ frame @ operator2mano
      // operator2mano right = [[0,0,-1],[-1,0,0],[0,1,0]], left = [[0,0,-1],[1,0,0],[0,-1,0]]
      const float sgn = left ? -1.f : 1.f;
#pragma unroll 3
      for (int j = 0; j < 21; ++j) {
        const float px = k[3 * j] - wx, py = k[3 * j + 1] - wy, pz = k[3 * j + 2] - wz;
        const float u = px * xx + py * xy + pz * xz;  // along x
        const float v = px * nx + py * ny + pz * nz;  // along normal
        const float w = px * zx + py * zy + pz * zz;  // along z
        k[3 * j] = -sgn * v;
        k[3 * j + 1] = sgn * w;
        k[3 * j + 2] = -u;
      }
      if (rot_out) {
        float* r = rot_out + (f0 + tid) * 9;
        r[0] = xx; r[1] = nx; r[2] = zx; r[3] = xy; r[4] = ny; r[5] = zy; r[6] = xz; r[7] = nz; r[8] = zz;
      }
    }
    __syncthreads();
    float* dst = out + f0 * 63;
    if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
      float4* d4 = reinterpret_cast<float4*>(dst);
      const float4* t4 = reinterpret_cast<const float4*>(tile);
      for (int i = tid; i < nfl / 4; i += kPreTile) d4[i] = t4[i];
      for (int i = (nfl / 4) * 4 + tid; i < nfl; i += kPreTile) dst[i] = tile[i];
    } else {
      for (int i = tid; i < nfl; i += kPreTile) dst[i] = tile[i];
    }
    __syncthreads();
  }
}

}  // namespace dexr

// ================================================================================================
// host side: handle, launches, C ABI
// ================================================================================================
using namespace dexr;

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// Every entry point that needs the robot's device current switches to it for the duration of the call only and puts
// the caller's device back on every exit path (a solve on an optimizer bound to cuda:1 must not move the calling
// thread's later `device="cuda"` allocations to that GPU).
struct DeviceGuard {
  int prev = -1;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device) {
    err = cudaGetDevice(&prev);
    if (err == cudaSuccess && prev != device) err = cudaSetDevice(device);
    else if (err == cudaSuccess) prev = -1;  // already current: nothing to restore
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define DEVICE_SCOPE(device)                                                                              \
  DeviceGuard _dev_guard(device);                                                                          \
  if (_dev_guard.err != cudaSuccess)                                                                       \
    return fail(DEXR_E_CUDA, "selecting device %d failed: %s", (int)(device), cudaGetErrorString(_dev_guard.err))

#define CUDA_TRY(expr)                                                                           \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return fail(DEXR_E_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

struct dexr_robot {
  int device = 0;
  int num_sms = 0;
  dexr_table_t* table_dev = nullptr;
  dexr_table_t host;  // header + small arrays used for validation / sizing
  dexr_launch_info_t last{};  // diagnostics only; guarded by info_mu (concurrent solves on one handle are allowed)
  std::mutex info_mu;
  // staging for dexr_solve_frames_host
  std::mutex mu;
  cudaStream_t streams[2] = {nullptr, nullptr};
  void* stage_dev[2] = {nullptr, nullptr};
  size_t stage_bytes = 0;
};

static int frames_max_tile(int lanes) { return lanes == 16 ? 64 : 32; }  // frames per ring stage (shared memory budget)
constexpr int kSeqNW = 8;       // warps per CTA (sequences kernel)

static int validate_table(const dexr_table_t* t) {
  if (t->magic != 0x31525844u) return fail(DEXR_E_INVALID, "robot table: bad magic 0x%08x", t->magic);
  if (t->nbytes != sizeof(dexr_table_t))
    return fail(DEXR_E_INVALID, "robot table: size %u does not match library (%zu)", t->nbytes, sizeof(dexr_table_t));
  if (t->dof < 1 || t->dof > DEXR_MAX_LANES) return fail(DEXR_E_INVALID, "robot table: dof %d out of range 1..32", t->dof);
  if (t->n_var < 1 || t->n_var > t->dof) return fail(DEXR_E_INVALID, "robot table: n_var %d out of range", t->n_var);
  if (t->n_fixed < 0 || t->n_fixed > t->dof) return fail(DEXR_E_INVALID, "robot table: n_fixed %d out of range", t->n_fixed);
  if (t->n_links < 1 || t->n_links > DEXR_MAX_LINKS) return fail(DEXR_E_INVALID, "robot table: n_links %d out of range", t->n_links);
  if (t->n_res < 1 || t->n_res > DEXR_MAX_RES) return fail(DEXR_E_INVALID, "robot table: n_res %d out of range", t->n_res);
  if (t->loss < 0 || t->loss > 2) return fail(DEXR_E_INVALID, "robot table: loss %d unknown", t->loss);
  if (t->n_rounds < 0 || t->n_rounds > 5) return fail(DEXR_E_INVALID, "robot table: n_rounds %d out of range", t->n_rounds);
  if (t->loss == DEXR_LOSS_DEXPILOT && (t->len_proj < 1 || t->len_proj > t->n_res || t->len_s1 > t->len_proj))
    return fail(DEXR_E_INVALID, "robot table: dexpilot projection sizes inconsistent");
  for (int k = 0; k < t->n_res; ++k) {
    if (t->res_task[k] < 0 || t->res_task[k] >= t->n_links || t->res_origin[k] >= t->n_links)
      return fail(DEXR_E_INVALID, "robot table: residual %d refers to an unknown link", k);
    if (t->res_human_task[k] < 0 || t->res_human_task[k] >= DEXR_NUM_KEYPOINTS ||
        t->res_human_origin[k] >= DEXR_NUM_KEYPOINTS)
      return fail(DEXR_E_INVALID, "robot table: residual %d human index out of range", k);
  }
  for (int k = 0; k < t->n_links; ++k)
    if (t->link_parent[k] >= t->dof) return fail(DEXR_E_INVALID, "robot table: link %d parent out of range", k);
  if (t->block_width != 0) {
    const int bw = t->block_width;
    if ((bw != 4 && bw != 8) || t->dof % bw != 0 || t->has_mimic || t->n_var != t->dof)
      return fail(DEXR_E_INVALID, "robot table: block_width %d inconsistent (dof %d, mimic %d)", bw, t->dof, t->has_mimic);
    for (int c = 0; c < t->dof; ++c) {  // ancestors must stay inside the lane window
      const uint32_t window = ((bw == 32 ? 0u : (1u << bw)) - 1u) << (c / bw * bw);
      if (t->anc_mask[c] & ~window) return fail(DEXR_E_INVALID, "robot table: block_width %d but joint %d has ancestors outside its window", bw, c);
    }
    for (int k = 0; k < t->n_res; ++k) {
      uint32_t m = t->link_anc_mask[t->res_task[k]] | (t->res_origin[k] >= 0 ? t->link_anc_mask[t->res_origin[k]] : 0u);
      if (m) {
        int first = __builtin_ctz(m) / bw, last = (31 - __builtin_clz(m)) / bw;
        if (first != last) return fail(DEXR_E_INVALID, "robot table: block_width %d but residual %d couples two windows", bw, k);
      }
    }
  }
  if (t->arrow != 0) {
    const int tr = t->arrow - 1;
    if (tr < 0 || tr > 8 || t->block_width != 0 || t->has_mimic || t->n_var != t->dof || t->dof <= 16 || tr >= t->dof)
      return fail(DEXR_E_INVALID, "robot table: arrow %d inconsistent (dof %d, mimic %d, block_width %d)", t->arrow, t->dof,
                  t->has_mimic, t->block_width);
    const uint32_t tmask = (1u << tr) - 1u;
    uint32_t finger_of[DEXR_MAX_LANES] = {0};  // lane -> mask of its finger's lanes
    int fingers = 0;
    for (int c = 0; c < tr; ++c)
      if (t->anc_mask[c] & ~tmask) return fail(DEXR_E_INVALID, "robot table: arrow trunk joint %d has an ancestor outside the trunk", c);
    for (int c = tr; c < t->dof; ++c) {
      const uint32_t chain = t->anc_mask[c] & ~tmask;  // includes c itself
      const int fb = __builtin_ctz(chain);
      if (fb == c) {
        const uint32_t span = t->desc_mask[c] | (1u << c);
        const int fw = 32 - __builtin_clz(span) - c;
        if (fw > 8 || ++fingers > 6 || span != ((fw == 32 ? 0u : (1u << fw)) - 1u) << c)
          return fail(DEXR_E_INVALID, "robot table: arrow finger at joint %d is not a contiguous run of <= 8 lanes (or > 6 fingers)", c);
        for (int i = c; i < c + fw; ++i) finger_of[i] = span;
      } else if (!((t->desc_mask[fb] >> c) & 1u)) {
        return fail(DEXR_E_INVALID, "robot table: arrow joint %d is not below its finger's first joint %d", c, fb);
      }
    }
    for (int c = tr; c < t->dof; ++c)
      if (!finger_of[c] || (t->anc_mask[c] & ~tmask & ~finger_of[c]))
        return fail(DEXR_E_INVALID, "robot table: arrow joint %d has ancestors in another finger", c);
    for (int k = 0; k < t->n_res; ++k) {
      uint32_t m = (t->link_anc_mask[t->res_task[k]] | (t->res_origin[k] >= 0 ? t->link_anc_mask[t->res_origin[k]] : 0u)) & ~tmask;
      if (m && (m & ~finger_of[__builtin_ctz(m)]))
        return fail(DEXR_E_INVALID, "robot table: arrow but residual %d couples two fingers", k);
    }
  }
  for (int c = 0; c < t->dof; ++c) {
    int n = 0;
    for (int k = 0; k < t->n_links; ++k) n += (t->link_parent[k] == c);
    if (n > DEXR_MAX_LINKS_PER_LANE)
      return fail(DEXR_E_INVALID, "robot table: %d objective links ride on joint %d (max %d)", n, c, DEXR_MAX_LINKS_PER_LANE);
  }
  return 0;
}

static int finish_create(dexr_robot* r, dexr_robot_t** out) {
  cudaDeviceProp prop;
  cudaError_t ce = cudaGetDeviceProperties(&prop, r->device);
  if (ce != cudaSuccess) {
    cudaFree(r->table_dev);
    delete r;
    return fail(DEXR_E_CUDA, "cudaGetDeviceProperties failed: %s", cudaGetErrorString(ce));
  }
  // arch-specific sm_90a code loads on compute capability 9.0 only
  if (prop.major != 9 || prop.minor != 0) {
    const int device = r->device;
    cudaFree(r->table_dev);
    delete r;
    return fail(DEXR_E_NODEVICE, "device %d is sm_%d%d; libdexr is built for sm_90a (H100) only", device, prop.major, prop.minor);
  }
  r->num_sms = prop.multiProcessorCount;
  *out = r;
  return 0;
}

extern "C" {

int dexr_version(void) { return DEXR_VERSION; }
#ifndef DEXR_BUILD_ID
#define DEXR_BUILD_ID "unstamped"
#endif
const char* dexr_build_id(void) { return DEXR_BUILD_ID; }
const char* dexr_last_error(void) { return g_err; }
size_t dexr_table_sizeof(void) { return sizeof(dexr_table_t); }
size_t dexr_params_sizeof(void) { return sizeof(dexr_params_t); }
size_t dexr_frames_sizeof(void) { return sizeof(dexr_frames_t); }
size_t dexr_sequences_sizeof(void) { return sizeof(dexr_sequences_t); }

void dexr_default_params(dexr_params_t* p) {
  p->huber_delta = 0.02f;
  p->norm_delta = 4e-3f;
  p->scaling = 1.0f;
  p->project_dist = 0.03f;
  p->escape_dist = 0.05f;
  p->eta1 = 1e-4f;
  p->eta2 = 3e-2f;
  p->lp_alpha = -1.0f;
  p->tol = 1e-5f;
  p->lambda0 = 1e-2f;
  p->max_iters = 64;
  p->clip_init = 0;
  p->preprocess = 0;
}

int dexr_robot_create(const dexr_table_t* table_host, int device, dexr_robot_t** out) {
  if (!table_host || !out) return fail(DEXR_E_INVALID, "dexr_robot_create: null argument");
  if (int e = validate_table(table_host)) return e;
  DEVICE_SCOPE(device);
  dexr_robot* r = new (std::nothrow) dexr_robot();
  if (!r) return fail(DEXR_E_INVALID, "out of host memory");
  r->device = device;
  r->host = *table_host;
  cudaError_t ce = cudaMalloc(&r->table_dev, sizeof(dexr_table_t));
  if (ce == cudaSuccess) ce = cudaMemcpy(r->table_dev, table_host, sizeof(dexr_table_t), cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) {
    if (r->table_dev) cudaFree(r->table_dev);
    delete r;
    return fail(DEXR_E_CUDA, "uploading the robot table failed: %s", cudaGetErrorString(ce));
  }
  return finish_create(r, out);
}

int dexr_robot_create_from_device(const void* table_dev, size_t nbytes, int device, dexr_robot_t** out) {
  if (!table_dev || !out) return fail(DEXR_E_INVALID, "dexr_robot_create_from_device: null argument");
  if (nbytes != sizeof(dexr_table_t)) return fail(DEXR_E_INVALID, "table size %zu != %zu", nbytes, sizeof(dexr_table_t));
  DEVICE_SCOPE(device);
  dexr_robot* r = new (std::nothrow) dexr_robot();
  if (!r) return fail(DEXR_E_INVALID, "out of host memory");
  r->device = device;
  cudaError_t ce = cudaMalloc(&r->table_dev, sizeof(dexr_table_t));
  if (ce == cudaSuccess) ce = cudaMemcpy(r->table_dev, table_dev, sizeof(dexr_table_t), cudaMemcpyDeviceToDevice);
  if (ce == cudaSuccess) ce = cudaMemcpy(&r->host, r->table_dev, sizeof(dexr_table_t), cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) {
    if (r->table_dev) cudaFree(r->table_dev);
    delete r;
    return fail(DEXR_E_CUDA, "adopting the device robot table failed: %s", cudaGetErrorString(ce));
  }
  if (int e = validate_table(&r->host)) {
    cudaFree(r->table_dev);
    delete r;
    return e;
  }
  return finish_create(r, out);
}

const void* dexr_robot_device_table(const dexr_robot_t* robot) { return robot ? robot->table_dev : nullptr; }

void dexr_robot_destroy(dexr_robot_t* robot) {
  if (!robot) return;
  DeviceGuard guard(robot->device);
  for (int i = 0; i < 2; ++i) {
    if (robot->streams[i]) cudaStreamDestroy(robot->streams[i]);
    if (robot->stage_dev[i]) cudaFree(robot->stage_dev[i]);
  }
  if (robot->table_dev) cudaFree(robot->table_dev);
  delete robot;
}

}  // extern "C"

static int check_params(const dexr_params_t* p) {
  if (!(p->huber_delta > 0.f)) return fail(DEXR_E_INVALID, "huber_delta must be > 0");
  if (!(p->norm_delta >= 0.f)) return fail(DEXR_E_INVALID, "norm_delta must be >= 0");
  if (p->max_iters < 1 || p->max_iters > 65535) return fail(DEXR_E_INVALID, "max_iters out of range");
  if (!(p->tol > 0.f) || !(p->lambda0 > 0.f)) return fail(DEXR_E_INVALID, "tol and lambda0 must be > 0");
  if (p->preprocess < 0 || p->preprocess > 2) return fail(DEXR_E_INVALID, "preprocess must be 0 (none), 1 (right hand) or 2 (left hand)");
  return 0;
}

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// DEXR_ARROW=0 forces the dense factorisation for tables that qualify for the arrow one.  Read per call (a getenv is
// nanoseconds against a launch) so that tests can compare the two inside one process.
static bool arrow_enabled() {
  const char* e = getenv("DEXR_ARROW");
  return !(e && atoi(e) == 0);
}

// Fill the kernel arguments of one robot group: tile size, ring layout, dynamic shared memory.  `slots` = CTAs the tiles are
// spread over.  Returns the dynamic shared memory the group needs.
template <int G, int NCW>
static int fill_frame_args(const dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, int slots, FrameArgs& a, int tile = 0) {
  const dexr_table_t& t = r->host;
  a = FrameArgs{};
  a.table = r->table_dev;
  a.prm = *prm;
  a.io = *io;
  a.B = B;
  a.dm = make_dims(t);
  a.in_row = io->keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * t.n_res;
  // Tile size: every CTA walks the tiles slot, slot + slots, ...; pick T so that the tile count lands just below a multiple of
  // the CTA count instead of always using the largest tile (B = 6144 on 132 SMs: 192 tiles of 32 leave 72 CTAs with one
  // tile and 60 with two -- 73 % efficiency; 256 tiles of 24 give all but 8 CTAs two).
  const long long per = (B + slots - 1) / slots;                                            // frames per CTA
  const int max_tile = frames_max_tile(G);
  const long long rounds = std::max<long long>(1, (per + max_tile - 1) / max_tile);
  int T = (int)std::min<long long>(max_tile, std::max<long long>(4, (per + rounds - 1) / rounds));
  T = round_up(T, 4);
  // A CTA solves NCW x (32 / G) frames at a time.  When its whole share fits one such round, rounding the tile up to the
  // bulk-copy granularity must not push it into a second, nearly empty round (Shadow, 2048 frames: 14 per CTA -> 16 on 15
  // warps): keep the exact count, the producer then stages the tile with plain loads.
  constexpr int kRound = NCW * (32 / G);
  if (per <= kRound && T > kRound) T = (int)per;
  if (tile > 0) T = std::min(tile, max_tile);  // mixed launches size the tiles of all groups together
  a.T = T;
  a.ntiles = (int)((B + T - 1) / T);
  auto aligned16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  // a tile starts on a 16-byte boundary of every input only when T is a multiple of 4 (252-byte keypoint rows): tiles of any
  // other size (exact one-round tiles) are staged with plain loads, their ragged last tile included
  a.use_bulk = (T & 3) == 0 && aligned16(io->keypoints ? io->keypoints : io->ref_value) && aligned16(io->last_qpos) &&
               (t.n_fixed == 0 || aligned16(io->fixed_qpos));
  a.off_in = 0;
  a.off_last = round_up(T * a.in_row * 4, 16);
  a.off_fixed = a.off_last + round_up(T * t.n_var * 4, 16);
  a.stage_bytes = a.off_fixed + round_up(T * std::max(t.n_fixed, 1) * 4, 16);
  a.ring_off = round_up((int)sizeof(SharedTable), 16);
  a.bar_off = a.ring_off + 2 * a.stage_bytes;
  a.scratch_off = round_up(a.bar_off + 4 * 8 + 2 * 4, 16);
  constexpr int GPW = 32 / G;
  return a.scratch_off + NCW * GPW * Scratch<G>::kFloats * 4;
}

template <int G, int BW, int NCW>
static int launch_frames(dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, cudaStream_t stream, int slots, int tile) {
  FrameArgs a;
  if (slots <= 0) slots = r->num_sms;  // one persistent CTA per SM; a mixed launch passes its own CTA count and tile size
  const int smem = fill_frame_args<G, NCW>(r, prm, io, B, slots, a, tile);
  auto kern = dexr_frames_kernel<G, BW, NCW>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = std::min(a.ntiles, slots);
  kern<<<grid, (NCW + 1) * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, (NCW + 1) * 32, smem, a.T, G, NCW, r->last.kernels_launched + 1};
  }
  return 0;
}

// Consumer warps per CTA for each solver kind (index = solver_kind()): the register file (64 K x 32 bit per SM, one CTA per
// SM) gives 128 registers per thread at 15 + 1 warps, 144 at 13 + 1, 168 at 11 + 1.  Measured on H100 SXM (400 W, 65 536
// frames per launch, 16 | 14 | 12 warps, ms): every solver kind is fastest with 16 warps despite the spills at 128
// registers -- Allegro vector (block) 0.265 | 0.290 | 0.305, LEAP DexPilot (dense 16) 1.77 | 1.86 | 1.80, Ability (dense 16,
// mimic) 1.52 | 1.67 | 1.75, Shadow position (arrow) 3.21 | 3.37 | 3.45, SVH (dense 32) 4.34 | 4.75 | 4.80.
// DEXR_FRAMES_WARPS="a,b,c,d" (16 | 14 | 12 per kind) overrides for A/B runs.
static const int* frames_warps() {
  static int w[4] = {16, 16, 16, 16};
  static const bool init = [] {
    if (const char* e = getenv("DEXR_FRAMES_WARPS")) {
      int v[4];
      if (sscanf(e, "%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3]) == 4)
        for (int i = 0; i < 4; ++i)
          if (v[i] == 16 || v[i] == 14 || v[i] == 12) w[i] = v[i];
    }
    return true;
  }();
  (void)init;
  return w;
}

template <int G, int BW>
static int launch_frames_warps(int warps, dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, cudaStream_t stream, int slots, int tile) {
  if (warps == 12) return launch_frames<G, BW, 11>(r, prm, io, B, stream, slots, tile);
  if (warps == 14) return launch_frames<G, BW, 13>(r, prm, io, B, stream, slots, tile);
  return launch_frames<G, BW, 15>(r, prm, io, B, stream, slots, tile);
}

static int launch_frames_kind(dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, cudaStream_t stream,
                              int slots = 0, int tile = 0) {
  const SolverKind k = solver_kind(r->host, arrow_enabled());
  const int warps = frames_warps()[k];
  return with_solver(k, [&](auto s) {
    return launch_frames_warps<decltype(s)::G, decltype(s)::BW>(warps, r, prm, io, B, stream, slots, tile);
  });
}

static int check_frames_io(const dexr_table_t& t, const dexr_frames_t* io, const dexr_params_t* prm) {
  if ((io->keypoints != nullptr) == (io->ref_value != nullptr))
    return fail(DEXR_E_INVALID, "exactly one of keypoints / ref_value must be given");
  if (prm->preprocess != 0 && !io->keypoints) return fail(DEXR_E_INVALID, "preprocess needs raw keypoints, not ref_value");
  if (!io->last_qpos || !io->qpos_out) return fail(DEXR_E_INVALID, "last_qpos and qpos_out are required");
  if (t.n_fixed > 0 && !io->fixed_qpos) return fail(DEXR_E_INVALID, "robot has %d fixed joints but fixed_qpos is NULL", t.n_fixed);
  return 0;
}

static int check_sequences_io(const dexr_table_t& t, const dexr_sequences_t* io, const dexr_params_t* prm) {
  if (!io->keypoints || !io->last_qpos || !io->robot_qpos_out) return fail(DEXR_E_INVALID, "keypoints, last_qpos, robot_qpos_out required");
  const bool use_filter = prm->lp_alpha >= 0.f && prm->lp_alpha <= 1.f;
  if (use_filter && (!io->filter_state || !io->filter_init)) return fail(DEXR_E_INVALID, "low-pass filter needs filter_state and filter_init");
  if (t.n_fixed > 0 && !io->fixed_qpos) return fail(DEXR_E_INVALID, "robot has %d fixed joints but fixed_qpos is NULL", t.n_fixed);
  return 0;
}

extern "C" int dexr_solve_frames_multi(const dexr_group_t* groups, int32_t num_groups, void* cuda_stream) {
  if (!groups) return fail(DEXR_E_INVALID, "dexr_solve_frames_multi: null argument");
  if (num_groups < 0 || num_groups > DEXR_MAX_GROUPS) return fail(DEXR_E_INVALID, "num_groups %d out of range 0..%d", num_groups, DEXR_MAX_GROUPS);
  constexpr int NCW = 15;
  MultiArgs m{};
  int smem = 0, device = -1, sms = 0;
  long long tiles = 0;
  dexr_robot* first = nullptr;
  for (int i = 0; i < num_groups; ++i) {
    const dexr_group_t& g = groups[i];
    if (!g.robot || !g.params) return fail(DEXR_E_INVALID, "group %d: null robot / params", i);
    if (g.num_frames < 0) return fail(DEXR_E_INVALID, "group %d: num_frames < 0", i);
    if (g.num_frames == 0) continue;
    if (int e = check_params(g.params)) return e;
    dexr_robot* r = const_cast<dexr_robot*>(g.robot);
    if (int e = check_frames_io(r->host, &g.io, g.params)) return e;
    if (device < 0) { device = r->device; sms = r->num_sms; first = r; }
    if (r->device != device) return fail(DEXR_E_INVALID, "group %d lives on device %d, group 0 on device %d: one launch, one device", i, r->device, device);
    const SolverKind k = solver_kind(r->host, arrow_enabled());
    FrameArgs& a = m.g[m.n_groups];
    const int need = kind_lanes(k) == 16 ? fill_frame_args<16, NCW>(r, g.params, &g.io, g.num_frames, sms, a)
                                         : fill_frame_args<32, NCW>(r, g.params, &g.io, g.num_frames, sms, a);
    smem = std::max(smem, need);
    m.kind[m.n_groups++] = k;
    tiles += a.ntiles;
  }
  if (m.n_groups == 0) return 0;
  DEVICE_SCOPE(device);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  // Two ways to run the groups:
  //  * streams (default): one standalone launch per group on library-owned side streams, forked from and joined back into
  //    the caller's stream with events.  Small groups have small grids and run side by side on different SMs, large ones
  //    overlap each other's tails.
  //  * persistent (DEXR_MULTI_MODE=persistent, read per call): ONE launch whose CTAs walk the groups
  //    (dexr_frames_multi_kernel).  Measured on H100 SXM (400 W) against the above -- six robots x n frames: n = 512: 0.58
  //    vs 0.27 ms, 2048: 0.80 vs 0.57, 16 384: 3.02 vs 2.81: the four solver bodies share one register allocation (748 B of
  //    spills against 32-128 B), and a CTA runs its groups one after the other where separate small grids run
  //    concurrently.  Kept for A/B runs; not the default.
  const char* mode_env = getenv("DEXR_MULTI_MODE");
  const bool persistent = mode_env && !strcmp(mode_env, "persistent");
  if (persistent) {
    auto kern = dexr_frames_multi_kernel<NCW>;
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = (int)std::min<long long>(tiles, sms);
    kern<<<grid, (NCW + 1) * 32, smem, stream>>>(m);
    CUDA_TRY(cudaGetLastError());
    std::lock_guard<std::mutex> lk(first->info_mu);
    first->last = dexr_launch_info_t{grid, (NCW + 1) * 32, smem, m.g[0].T, 0, NCW, first->last.kernels_launched + 1};
    return 0;
  }
  // fork / join.  The side streams and events belong to the library (one set per device, created on first use); a mutex
  // serialises their use by concurrent callers.
  struct Side { cudaStream_t s[DEXR_MAX_GROUPS] = {}; cudaEvent_t done[DEXR_MAX_GROUPS] = {}; cudaEvent_t fork = nullptr; };
  static std::mutex side_mu;
  static Side side[16];
  if (device >= 16) return fail(DEXR_E_INVALID, "device index %d beyond the side-stream table", device);
  std::lock_guard<std::mutex> lock(side_mu);
  Side& sd = side[device];
  if (!sd.fork) CUDA_TRY(cudaEventCreateWithFlags(&sd.fork, cudaEventDisableTiming));
  CUDA_TRY(cudaEventRecord(sd.fork, stream));
  // Sizing the CTAs of all groups TOGETHER.  A CTA takes a whole SM (registers), so the CTAs of the concurrent kernels queue
  // for SMs, and a CTA solves `round` = warps x frames-per-warp frames at a time.  A group that spreads over all SMs on its
  // own (what a lone launch does) gives each CTA a thin tile that still costs whole rounds -- six robots x 2048 frames: 768
  // CTAs, the 32-lane ones with 16 frames on 15 warps = two rounds, the second with one frame.  Instead, with
  //   R = sum over groups of ceil(frames / round)   (CTA-rounds of work):
  //   R <= SMs:      one wave; tiles shrunk by the common factor R / SMs so that every SM gets a CTA;
  //   R < 8 SMs:     every CTA gets r = max(1, R / (4 SMs)) whole rounds and there are as many CTAs as that takes (about
  //                  four waves; the hardware's CTA scheduler balances them over the SMs);
  //   otherwise:     one persistent CTA per SM and group as in a lone launch (enough work per SM that the dynamic frame
  //                  queue inside a CTA balances better than many short CTAs);
  //   always:        groups are launched slowest solver first (32-lane dense, arrow, 16-lane dense, block diagonal), so the
  //                  long CTAs are dispatched first and the short ones fill the tail.
  // Measured on H100 SXM (400 W), six robots x n frames, ms per call, lone-launch sizing in the given order -> this:
  // n = 512: 0.53 -> 0.27, 2048: 0.62 -> 0.57, 16 384: 2.82 -> 2.81.
  // DEXR_MULTI_SLOTS=spread (read per call) restores the lone-launch sizing and the given order for A/B runs.
  const char* slots_env = getenv("DEXR_MULTI_SLOTS");
  const bool packed = !(slots_env && !strcmp(slots_env, "spread")) && m.n_groups > 1;
  struct Plan { int group, kind, slots, tile; };
  Plan plan[DEXR_MAX_GROUPS];
  int n_plan = 0;
  long long R = 0;
  auto round_of = [](int kind) { return (frames_warps()[kind] - 1) * (32 / kind_lanes(kind)); };
  for (int i = 0; i < num_groups; ++i) {
    if (groups[i].num_frames == 0) continue;
    const int k = solver_kind(groups[i].robot->host, arrow_enabled());
    plan[n_plan++] = Plan{i, k, 0, 0};
    R += (groups[i].num_frames + round_of(k) - 1) / round_of(k);
  }
  // tunables for A/B sweeps (read per call): CTA waves aimed at, and the work per SM (in rounds) from which every group goes
  // back to one persistent CTA per SM
  auto env_int = [](const char* name, int dflt) { const char* e = getenv(name); return e && atoi(e) > 0 ? atoi(e) : dflt; };
  const int waves = env_int("DEXR_MULTI_WAVES", 4), spread_at = env_int("DEXR_MULTI_SPREAD_AT", 8);
  if (packed && R < (long long)spread_at * sms) {
    const long long r = std::max<long long>(1, R / ((long long)waves * sms));
    for (int j = 0; j < n_plan; ++j) {
      Plan& p = plan[j];
      const long long B = groups[p.group].num_frames;
      const int S = round_of(p.kind), max_tile = frames_max_tile(kind_lanes(p.kind));
      long long per = R <= sms ? std::max<long long>(1, (S * R + sms - 1) / sms) : r * S;  // frames per CTA
      if (per <= max_tile) {                                 // one tile per CTA
        p.tile = (int)(per > S ? (per & ~3LL) : per);  // one round: exactly the frames the warps hold (plain loads if not 4 | tile)
        p.slots = (int)std::min<long long>((B + p.tile - 1) / p.tile, 1 << 20);
      } else {
        p.slots = (int)((B + per - 1) / per);
      }
    }
  }
  if (packed) std::stable_sort(plan, plan + n_plan, [](const Plan& x, const Plan& y) { return x.kind > y.kind; });
  // A failure in the middle must not leave kernels of this call running behind the caller's stream: every side stream that
  // was forked is joined whatever happens after it, and the first error is reported at the end.
  int rc = 0;
  for (int gi = 0; gi < n_plan && rc == 0; ++gi) {
    const dexr_group_t& g = groups[plan[gi].group];
    if (!sd.s[gi]) {
      CUDA_TRY(cudaStreamCreateWithFlags(&sd.s[gi], cudaStreamNonBlocking));
      CUDA_TRY(cudaEventCreateWithFlags(&sd.done[gi], cudaEventDisableTiming));
    }
    cudaError_t ce = cudaStreamWaitEvent(sd.s[gi], sd.fork, 0);
    if (ce == cudaSuccess)
      rc = launch_frames_kind(const_cast<dexr_robot*>(g.robot), g.params, &g.io, g.num_frames, sd.s[gi], plan[gi].slots, plan[gi].tile);
    if (ce == cudaSuccess) ce = cudaEventRecord(sd.done[gi], sd.s[gi]);
    if (ce == cudaSuccess) ce = cudaStreamWaitEvent(stream, sd.done[gi], 0);
    if (ce != cudaSuccess && rc == 0) rc = fail(DEXR_E_CUDA, "dexr_solve_frames_multi: group %d: %s", plan[gi].group, cudaGetErrorString(ce));
  }
  return rc;
}

extern "C" int dexr_solve_frames(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_frames_t* io,
                                 int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_frames: null argument");
  if (num_frames < 0) return fail(DEXR_E_INVALID, "num_frames < 0");
  if (num_frames == 0) return 0;
  if (int e = check_params(params)) return e;
  const dexr_table_t& t = robot->host;
  if (int e = check_frames_io(t, io, params)) return e;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return launch_frames_kind(r, params, io, num_frames, stream);
}

template <int G, int BW>
static int launch_sequences(dexr_robot* r, const dexr_params_t* prm, const dexr_sequences_t* io, long long S, int steps,
                            cudaStream_t stream) {
  const dexr_table_t& t = r->host;
  SeqArgs a{};
  a.table = r->table_dev;
  a.prm = sequence_params(*prm);
  a.io = *io;
  a.S = S;
  a.steps = steps;
  a.dm = make_dims(t);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int groups = kSeqNW * GPW;
  const int smem = a.scratch_off + groups * Scratch<G>::kStreamFloats * 4;
  auto kern = dexr_sequences_kernel<G, BW, kSeqNW>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // A stream is serial in time and latency bound, so streams are spread over as many warps and SMs as there are: while one
  // warp per stream fits into one wave of CTAs (S <= SMs x warps per CTA), a warp carries ONE stream (the second group of a
  // 16-lane solver idles); beyond that two 16-lane streams share a warp.  One CTA per SM, two when streams are plentiful.
  const long long warps_one_wave = (long long)r->num_sms * kSeqNW;
  a.spw = (GPW > 1 && S > warps_one_wave) ? GPW : 1;
  static const int spw_env = [] { const char* e = getenv("DEXR_SEQ_PAIR"); return e ? atoi(e) : -1; }();  // A/B: 1 = always pair
  if (spw_env == 1) a.spw = GPW;
  const char* duo_env = getenv("DEXR_SEQ_DUO");  // 0 = off (read per call: tests compare the two modes in one process)
  a.duo = (G == 16 && a.spw == 1 && !(duo_env && atoi(duo_env) == 0)) ? 1 : 0;
  const long long per_cta = (long long)kSeqNW * a.spw;
  const long long ctas = std::max<long long>(1, (S + a.spw - 1) / a.spw);  // at least one warp's worth of streams per CTA
  int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * (S >= (long long)r->num_sms * per_cta * 2 ? 2 : 1));
  kern<<<grid, kSeqNW * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kSeqNW * 32, smem, 0, G, kSeqNW, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_solve_sequences(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                                    int64_t num_streams, int64_t num_steps, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_sequences: null argument");
  if (num_streams < 0 || num_steps < 0 || num_steps > INT32_MAX) return fail(DEXR_E_INVALID, "bad sizes");
  if (num_streams == 0 || num_steps == 0) return 0;
  if (int e = check_params(params)) return e;
  if (int e = check_sequences_io(robot->host, io, params)) return e;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return with_solver(solver_kind(r->host, arrow_enabled()), [&](auto s) {
    return launch_sequences<decltype(s)::G, decltype(s)::BW>(r, params, io, num_streams, (int)num_steps, stream);
  });
}

extern "C" {

int dexr_preprocess_keypoints(const float* raw, float* out, float* wrist_rot_out, int hand_type, int64_t num_frames,
                              int device, void* cuda_stream) {
  if (!raw || !out) return fail(DEXR_E_INVALID, "dexr_preprocess_keypoints: null argument");
  if (num_frames < 0 || (hand_type != 0 && hand_type != 1)) return fail(DEXR_E_INVALID, "bad num_frames / hand_type");
  if (num_frames == 0) return 0;
  DEVICE_SCOPE(device);
  int sms = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const long long tiles = (num_frames + kPreTile - 1) / kPreTile;
  const int grid = (int)std::min<long long>(tiles, (long long)sms * 8);
  dexr_preprocess_kernel<<<grid, kPreTile, 0, static_cast<cudaStream_t>(cuda_stream)>>>(raw, out, wrist_rot_out, hand_type,
                                                                                          (long long)num_frames);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int dexr_get_launch_info(const dexr_robot_t* robot, dexr_launch_info_t* out) {
  if (!robot || !out) return fail(DEXR_E_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(const_cast<dexr_robot*>(robot)->info_mu);
  *out = robot->last;
  return 0;
}

// Host-buffer entry: chunked, two internal streams so that chunk i+1's H2D overlaps chunk i's solve
// and chunk i-1's D2H.  Pointers in `io_host` are host pointers (pinned for true overlap).
int dexr_solve_frames_host(dexr_robot_t* robot, const dexr_params_t* params, const dexr_frames_t* h, int64_t B) {
  if (!robot || !params || !h) return fail(DEXR_E_INVALID, "dexr_solve_frames_host: null argument");
  if (B < 0) return fail(DEXR_E_INVALID, "num_frames < 0");
  if (B == 0) return 0;
  const dexr_table_t& t = robot->host;
  if (int e = check_frames_io(t, h, params)) return e;
  std::lock_guard<std::mutex> lock(robot->mu);
  DEVICE_SCOPE(robot->device);
  const int in_row = h->keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * t.n_res;
  if (!robot->streams[0]) CUDA_TRY(cudaStreamCreateWithFlags(&robot->streams[0], cudaStreamNonBlocking));
  // Zero-copy fast path: when every buffer is page-locked host memory (cudaHostAlloc / cudaHostRegister, e.g.
  // torch pin_memory()), the kernel reads and writes it directly -- the producer warp's bulk copies pull the
  // input tiles over PCIe straight into shared memory while the consumers compute, results go back with
  // 64-byte stores: one launch, no staging buffers, copy fully overlapped with the solve.
  // (DexPilot flags are read-modify-written byte-wise: that case keeps the staged path.)
  static const bool zero_copy = [] { const char* e = getenv("DEXR_HOST_ZEROCOPY"); return !(e && atoi(e) == 0); }();
  if (zero_copy && !h->projected) {
    bool ok = true;
    dexr_frames_t d = *h;
    auto map = [&](const void* host, const void** dev) {
      if (!host) { *dev = nullptr; return; }
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, host) != cudaSuccess) { cudaGetLastError(); ok = false; return; }
      if (a.type != cudaMemoryTypeHost || !a.devicePointer) { ok = false; return; }
      *dev = a.devicePointer;
    };
    map(h->keypoints, (const void**)&d.keypoints);
    map(h->ref_value, (const void**)&d.ref_value);
    map(h->fixed_qpos, (const void**)&d.fixed_qpos);
    map(h->last_qpos, (const void**)&d.last_qpos);
    map(h->qpos_out, (const void**)&d.qpos_out);
    map(h->robot_qpos_out, (const void**)&d.robot_qpos_out);
    map(h->status_out, (const void**)&d.status_out);
    map(h->cost_out, (const void**)&d.cost_out);
    map(h->damping_io, (const void**)&d.damping_io);
    if (ok) {
      if (int e = dexr_solve_frames(robot, params, &d, B, robot->streams[0])) return e;
      CUDA_TRY(cudaStreamSynchronize(robot->streams[0]));
      return 0;
    }
  }
  // per-frame device bytes, every sub-array padded so that chunk bases stay 16-byte aligned
  const size_t row_in = in_row * 4, row_last = t.n_var * 4, row_fixed = t.n_fixed * 4, row_proj = t.len_proj,
               row_q = t.n_var * 4, row_rq = h->robot_qpos_out ? t.dof * 4 : 0, row_st = h->status_out ? 4 : 0,
               row_c = h->cost_out ? 4 : 0, row_dmp = h->damping_io ? 4 : 0;
  // chunks per call: enough to overlap copies with the solve, few enough that each launch still fills the GPU
  static const int n_chunks_env = [] { const char* e = getenv("DEXR_HOST_CHUNKS"); return e ? std::max(1, atoi(e)) : 0; }();
  const int n_chunks = n_chunks_env ? n_chunks_env : 4;
  const int64_t chunk = std::min<int64_t>(B, std::max<int64_t>(4096, round_up((int)std::min<int64_t>((B + n_chunks - 1) / n_chunks, 1 << 20), 64)));
  auto pad = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t need = pad(chunk * row_in) + pad(chunk * row_last) + pad(chunk * row_fixed) + pad(chunk * row_proj) +
                      pad(chunk * row_q) + pad(chunk * row_rq) + pad(chunk * row_st) + pad(chunk * row_c) + pad(chunk * row_dmp);
  for (int i = 0; i < 2; ++i)
    if (!robot->streams[i]) CUDA_TRY(cudaStreamCreateWithFlags(&robot->streams[i], cudaStreamNonBlocking));
  if (robot->stage_bytes < need) {  // grow both staging buffers, or leave the handle with none (never a stale size)
    for (int i = 0; i < 2; ++i) {
      if (robot->stage_dev[i]) cudaFree(robot->stage_dev[i]);
      robot->stage_dev[i] = nullptr;
    }
    robot->stage_bytes = 0;
    for (int i = 0; i < 2; ++i) {
      cudaError_t ce = cudaMalloc(&robot->stage_dev[i], need);
      if (ce != cudaSuccess) {
        for (int j = 0; j < 2; ++j) {
          if (robot->stage_dev[j]) cudaFree(robot->stage_dev[j]);
          robot->stage_dev[j] = nullptr;
        }
        return fail(DEXR_E_CUDA, "allocating %zu staging bytes failed: %s", need, cudaGetErrorString(ce));
      }
    }
    robot->stage_bytes = need;
  }
  // From the first enqueue on, an error must not return while copies / kernels are still in flight on the two internal
  // streams (they write into the caller's host buffers): run the pipeline in a lambda, drain both streams, then report.
  auto pipeline = [&]() -> int {
  int ci = 0;
  for (int64_t f0 = 0; f0 < B; f0 += chunk, ci ^= 1) {
    const int64_t n = std::min<int64_t>(chunk, B - f0);
    cudaStream_t s = robot->streams[ci];
    unsigned char* base = static_cast<unsigned char*>(robot->stage_dev[ci]);
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base + off; off += pad(bytes); return p; };
    float* d_in = reinterpret_cast<float*>(take(chunk * row_in));
    float* d_last = reinterpret_cast<float*>(take(chunk * row_last));
    float* d_fixed = reinterpret_cast<float*>(take(chunk * row_fixed));
    uint8_t* d_proj = reinterpret_cast<uint8_t*>(take(chunk * row_proj));
    float* d_q = reinterpret_cast<float*>(take(chunk * row_q));
    float* d_rq = reinterpret_cast<float*>(take(chunk * row_rq));
    int32_t* d_st = reinterpret_cast<int32_t*>(take(chunk * row_st));
    float* d_c = reinterpret_cast<float*>(take(chunk * row_c));
    float* d_dmp = reinterpret_cast<float*>(take(chunk * row_dmp));
    const float* h_in = h->keypoints ? h->keypoints : h->ref_value;
    CUDA_TRY(cudaMemcpyAsync(d_in, h_in + f0 * in_row, n * row_in, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_last, h->last_qpos + f0 * t.n_var, n * row_last, cudaMemcpyHostToDevice, s));
    if (t.n_fixed) CUDA_TRY(cudaMemcpyAsync(d_fixed, h->fixed_qpos + f0 * t.n_fixed, n * row_fixed, cudaMemcpyHostToDevice, s));
    const bool proj = h->projected && t.len_proj > 0;
    if (proj) CUDA_TRY(cudaMemcpyAsync(d_proj, h->projected + f0 * t.len_proj, n * row_proj, cudaMemcpyHostToDevice, s));
    if (h->damping_io) CUDA_TRY(cudaMemcpyAsync(d_dmp, h->damping_io + f0, n * row_dmp, cudaMemcpyHostToDevice, s));
    dexr_frames_t d{};
    d.damping_io = h->damping_io ? d_dmp : nullptr;
    d.keypoints = h->keypoints ? d_in : nullptr;
    d.ref_value = h->keypoints ? nullptr : d_in;
    d.last_qpos = d_last;
    d.fixed_qpos = t.n_fixed ? d_fixed : nullptr;
    d.projected = proj ? d_proj : nullptr;
    d.qpos_out = d_q;
    d.robot_qpos_out = h->robot_qpos_out ? d_rq : nullptr;
    d.status_out = h->status_out ? d_st : nullptr;
    d.cost_out = h->cost_out ? d_c : nullptr;
    if (int e = dexr_solve_frames(robot, params, &d, n, s)) return e;
    CUDA_TRY(cudaMemcpyAsync(h->qpos_out + f0 * t.n_var, d_q, n * row_q, cudaMemcpyDeviceToHost, s));
    if (h->robot_qpos_out) CUDA_TRY(cudaMemcpyAsync(h->robot_qpos_out + f0 * t.dof, d_rq, n * row_rq, cudaMemcpyDeviceToHost, s));
    if (h->status_out) CUDA_TRY(cudaMemcpyAsync(h->status_out + f0, d_st, n * row_st, cudaMemcpyDeviceToHost, s));
    if (h->cost_out) CUDA_TRY(cudaMemcpyAsync(h->cost_out + f0, d_c, n * row_c, cudaMemcpyDeviceToHost, s));
    if (h->damping_io) CUDA_TRY(cudaMemcpyAsync(h->damping_io + f0, d_dmp, n * row_dmp, cudaMemcpyDeviceToHost, s));
    if (proj) CUDA_TRY(cudaMemcpyAsync(h->projected + f0 * t.len_proj, d_proj, n * row_proj, cudaMemcpyDeviceToHost, s));
    // the staging buffer of this stream is reused two chunks later: same stream => ordered
  }
  return 0;
  };
  const int rc = pipeline();
  const cudaError_t s0 = cudaStreamSynchronize(robot->streams[0]);
  const cudaError_t s1 = cudaStreamSynchronize(robot->streams[1]);
  if (rc != 0) return rc;  // g_err holds the first failure
  if (s0 != cudaSuccess || s1 != cudaSuccess)
    return fail(DEXR_E_CUDA, "staged host pipeline failed: %s", cudaGetErrorString(s0 != cudaSuccess ? s0 : s1));
  return 0;
}

}  // extern "C"
