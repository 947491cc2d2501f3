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
// The tile queue of one frames launch (FrameArgs::queue): tiles handed out beyond every CTA's first tile, and the CTAs
// that are done with it.  The launch's last CTA zeroes it again.  Library-owned slots, one launch at a time per slot
// (dexr_robot::queue_dev).
struct QueueSlot {
  unsigned int next, done;
};

constexpr int kMaxLevels = 6;

struct FrameArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_frames_t io;
  long long B;
  int T;          // frames per full tile (multiple of 4, except the exact one-round tiles)
  int ntiles;     // full tiles: the static schedule's count
  int stages;     // input ring depth
  int min_chunk;  // queue: smallest tile handed out as the queue runs dry (= T: tiles never shrink)
  QueueSlot* queue;  // nullptr: static striding (tiles first_tile, first_tile + gridDim.x, ...)
  int n_levels;      // queue schedule after the grid's first tiles: lv_tiles[j] tiles of lv_size[j] frames, j = 0, 1, ...
  int lv_tiles[kMaxLevels], lv_size[kMaxLevels];
  unsigned long long* timeline;  // DEXR_EXP_TIMELINE builds: event buffer (frames_timeline.py); otherwise unused
  int use_bulk;   // inputs 16-byte aligned -> cp.async.bulk for full tiles
  int in_row;     // floats per frame of the kp/ref input (63 or 3m)
  Dims dm;
  int off_in, off_last, off_fixed, stage_bytes;  // ring stage layout (bytes)
  int ring_off, bar_off, scratch_off;            // dynamic smem layout (bytes)
};

// Experiment build DEXR_EXP_TIMELINE: the frames kernel records when each of its warps waits and works, into a buffer the
// caller passes with dexr_exp_timeline() (tools/frames_timeline.py reads it).  Layout, 64-bit words: an event count per
// (CTA, warp) for kTlCtas x 32 warps, then kTlEvents events of 4 words per (CTA, warp): {kind << 32 | x, y, t0, t1} with
// %globaltimer nanoseconds.  Kinds: 0 warp span (entry, exit), 1 consumer frame claim (x = first frame, y = frames),
// 2 consumer wait on a stage (x = tile's first frame, y = frames), 3 producer wait for a free stage, 4 producer tile claim
// (x = first frame, y = frames), 5 consumer prologue (entry to table loaded and solver set up), 6 consumer warp's totals at its
// exit (x = outer iterations its solver ran, y = frames it solved).  The default build records nothing.
constexpr int kTlCtas = 256, kTlEvents = 128;
struct Timeline {
#ifdef DEXR_EXP_TIMELINE
  unsigned long long* w = nullptr;
  unsigned long long* cnt = nullptr;
  int n = 0;
  __device__ __forceinline__ Timeline(unsigned long long* buf, int warp) {
    if (buf && blockIdx.x < kTlCtas && threadIdx.x % 32 == 0) {
      const int slot = blockIdx.x * 32 + warp;
      cnt = buf + slot;
      w = buf + kTlCtas * 32 + (size_t)slot * kTlEvents * 4;
    }
  }
  __device__ __forceinline__ static unsigned long long now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
  }
  __device__ __forceinline__ void event(int kind, long long x, long long y, unsigned long long t0, unsigned long long t1) {
    if (w && n < kTlEvents) {
      w[4 * n] = ((unsigned long long)kind << 32) | (unsigned int)x;
      w[4 * n + 1] = (unsigned long long)y;
      w[4 * n + 2] = t0;
      w[4 * n + 3] = t1;
      ++n;
    }
  }
  __device__ __forceinline__ void close() {
    if (cnt) *cnt = (unsigned long long)n;
  }
#else
  __device__ __forceinline__ Timeline(unsigned long long*, int) {}
  __device__ __forceinline__ static unsigned long long now() { return 0; }
  __device__ __forceinline__ void event(int, long long, long long, unsigned long long, unsigned long long) {}
  __device__ __forceinline__ void close() {}
#endif
};
#ifdef DEXR_EXP_TIMELINE
static unsigned long long* g_timeline = nullptr;  // set by dexr_exp_timeline(), passed to every frames launch
#endif

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
// Programmatic dependent launch (launch_frames_kernel): the next kernel of the stream may be launched as soon as every CTA
// of this one has started, so its CTAs take the SMs this launch's CTAs leave and run their set-up while the rest of this
// launch finishes.  grid_dep_wait() returns once the previous kernel of the stream has completed and its writes are
// visible; the frames kernel reads nothing the previous kernel may write before it (the robot table is only written by
// copies, never by a kernel).  Both are no-ops in a kernel not launched that way.
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// One robot group, executed by one CTA.  Its first tile is `first_tile`; after that it takes the tiles
// `first_tile + gridDim.x, first_tile + 2 gridDim.x, ...` (static striding, a.queue == nullptr), or claims tiles from the
// launch's queue (a.queue), which hands out the frames beyond the grid's first tiles in tiles that shrink as it runs dry.
// The producer writes each tile's first frame and size next to its stage; a size of 0 tells the consumers that the group
// is done.  Both the single-robot kernel and the mixed-robot kernel (several groups back to back inside one launch) run
// this body; it starts with a CTA-wide barrier and leaves every barrier phase complete, so it can be called repeatedly with
// different tables / template parameters.
template <int G, int BW, int NCW>
__device__ __forceinline__ void frames_group(const FrameArgs& a, int first_tile) {
  unsigned char* const smem = dsmem;
  SharedTable* st = reinterpret_cast<SharedTable*>(smem);
  unsigned char* ring = smem + a.ring_off;
  const int S = a.stages;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + a.bar_off);
  uint64_t* empty = full + S;
  long long* tile_f0 = reinterpret_cast<long long*>(empty + S);
  int* next = reinterpret_cast<int*>(tile_f0 + S);
  int* tile_n = next + S;

  // warp-uniform by construction: tells the compiler that the role split below never splits a warp
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  Timeline tl(a.timeline, warp);
  const unsigned long long t_entry = Timeline::now();

  __syncthreads();  // (mixed launches: every warp is done with the previous group's table, ring and barriers)
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NCW);
    }
    mbar_fence_init();
  }
  __syncthreads();

  const bool by_kp = a.io.keypoints != nullptr;
  const float* g_in = by_kp ? a.io.keypoints : a.io.ref_value;

  if (warp == NCW) {
    // ===================== producer: stage tiles HBM -> shared memory =====================
    // frames the grid's first tiles cover: the queue hands out the rest
    const long long head = min(a.B, (long long)gridDim.x * a.T);
    long long f0 = (long long)first_tile * a.T;
    int count = (int)max(0LL, min((long long)a.T, a.B - f0));
    grid_dep_wait();  // (the inputs and the queue)
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0;; ++it) {
      if (it >= S) {
        const unsigned long long t0 = Timeline::now();
        mbar_wait(&empty[stage], phase ^ 1u);
        tl.event(3, 0, 0, t0, Timeline::now());
      }
      if (lane == 0) {
        tile_f0[stage] = f0;
        tile_n[stage] = count;
        next[stage] = 0;
      }
      if (count == 0) {  // end of the group: every consumer reads the size 0 and leaves
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[stage]);
        break;
      }
      unsigned char* sb = ring + stage * a.stage_bytes;
      float* s_in = reinterpret_cast<float*>(sb + a.off_in);
      float* s_last = reinterpret_cast<float*>(sb + a.off_last);
      float* s_fixed = reinterpret_cast<float*>(sb + a.off_fixed);
      const float* gi = g_in + f0 * a.in_row;
      const float* gl = a.io.last_qpos + f0 * a.dm.n_var;
      const float* gf = a.dm.n_fixed > 0 ? a.io.fixed_qpos + f0 * a.dm.n_fixed : nullptr;
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
      if (++stage == S) {
        stage = 0;
        phase ^= 1u;
      }
      // the next tile
      if (!a.queue) {
        f0 += (long long)gridDim.x * a.T;
        count = (int)max(0LL, min((long long)a.T, a.B - f0));
      } else {
        // One atomicAdd per claim (a compare-and-swap loop on the frame count stalls once every CTA claims at the same
        // time, as they do while the queue runs dry): the k-th claim of the launch gets the k-th tile of a fixed schedule
        // (FrameArgs::lv_*), full tiles first, then tiles that shrink level by level (see plan_queue).
        if (lane == 0) {
          const unsigned long long t0 = Timeline::now();
          int k = (int)atomicAdd(&a.queue->next, 1u);
          long long f = head;
          count = 0;
          for (int j = 0; j < a.n_levels; ++j) {
            if (k < a.lv_tiles[j]) {
              f0 = f + (long long)k * a.lv_size[j];
              count = (int)min((long long)a.lv_size[j], a.B - f0);
              break;
            }
            k -= a.lv_tiles[j];
            f += (long long)a.lv_tiles[j] * a.lv_size[j];
          }
          if (count) tl.event(4, f0, count, t0, Timeline::now());
        }
        f0 = __shfl_sync(0xffffffffu, f0, 0);
        count = __shfl_sync(0xffffffffu, count, 0);
      }
    }
    if (a.queue && lane == 0) {
      // This CTA's last claim found the queue empty.  The last CTA to get here knows that no CTA of the launch will read
      // the queue again and zeroes it for the next launch that takes this slot.
      __threadfence();
      if (atomicAdd(&a.queue->done, 1u) == gridDim.x - 1) {
        a.queue->next = 0;
        a.queue->done = 0;
      }
    }
  } else {
    // ===================== consumers: one frame per group of G lanes =========================
    // The consumers load the table while the producer's first tiles are in flight, and wait for each other only (named
    // barrier 1).  Every array of the table has at most 32 entries, so threads of warp 0 copy all of it and the producer
    // warp has no part in load_shared_table.
    load_shared_table(*st, a.table, pass_slot_width<BW>());
    grid_dep_wait();  // (the damping words and every output)
    asm volatile("bar.sync 1, %0;" ::"r"(NCW * 32) : "memory");
    constexpr int GPW = 32 / G;
    const int gid = warp * GPW + (lane / G);
    Solver<G, BW> sv;
    sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * Scratch<G, BW>::kFloats * 4), a.prm, lane);
    tl.event(5, 0, 0, t_entry, Timeline::now());

    long long solved = 0;  // (timeline builds: frames this warp solved)
    for (int it = 0;; ++it) {
      const int stage = it % S;
      const unsigned long long t_wait = Timeline::now();
      mbar_wait(&full[stage], (uint32_t)(it / S) & 1u);
      // the stage's first frame and size are reread from shared memory where they are used: nothing lives in registers
      // across solve_frame that the static schedule did not keep there
      const volatile long long* v_f0 = tile_f0 + stage;
      const volatile int* v_n = tile_n + stage;
      tl.event(2, *v_f0, *v_n, t_wait, Timeline::now());
      if (*v_n == 0) {  // the group is done; arriving keeps the stage's barrier phases complete for the next group
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        break;
      }
      const unsigned char* sb = ring + stage * a.stage_bytes;
      const float* s_in = reinterpret_cast<const float*>(sb + a.off_in);
      const float* s_last = reinterpret_cast<const float*>(sb + a.off_last);
      const float* s_fixed = reinterpret_cast<const float*>(sb + a.off_fixed);
      while (true) {
        int base = 0;
        if (lane == 0) base = atomicAdd(&next[stage], GPW);
        base = __shfl_sync(0xffffffffu, base, 0);
        const int count = *v_n;
        if (base >= count) break;
        const int idx = base + (lane / G);
        const bool active = idx < count;
        const int ci = active ? idx : base;
        const long long f = *v_f0 + ci;
        FrameInputs in;
        in.kp = by_kp ? s_in + ci * a.in_row : nullptr;
        in.ref = by_kp ? nullptr : s_in + ci * a.in_row;
        in.last = s_last + ci * a.dm.n_var;
        in.fixed = s_fixed + ci * a.dm.n_fixed;
        in.projected = a.io.projected ? a.io.projected + f * a.dm.len_proj : nullptr;
        const unsigned long long t0 = Timeline::now();
        solve_frame(sv, in, a.io, a.dm, f, active);
        tl.event(1, f - ci + base, min(GPW, *v_n - base), t0, Timeline::now());
#ifdef DEXR_EXP_TIMELINE
        solved += min(GPW, *v_n - base);
#endif
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
    }
    tl.event(6, sv.issued, solved, t_entry, Timeline::now());
  }
  tl.event(0, blockIdx.x, warp, t_entry, Timeline::now());
  tl.close();
}

template <int G, int BW, int NCW>
__global__ void __launch_bounds__((NCW + 1) * 32, 1) dexr_frames_kernel(const FrameArgs a) {
  grid_dep_launch();
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
  const uint32_t scratch_off = (uint32_t)(a.scratch_off + gid * Scratch<G, BW>::kStreamFloats * 4);
  float* kpbuf = reinterpret_cast<float*>(smem + scratch_off) + Scratch<G, BW>::kFloats;  // 63 floats: current keypoints
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

// dexr_solve_sequences_tape: dexr_sequences_kernel line for line, with solve_stream's recording switched on.  (A body shared
// through an inline function changes how ptxas orders the filter test of dexr_sequences_kernel; this twin leaves that
// kernel's machine code as it was.)
template <int G, int BW, int NW>
__global__ void __launch_bounds__(NW * 32, 1) dexr_sequences_tape_kernel(const SeqArgs a, const dexr_sequences_tape_t tape) {
  unsigned char* const smem = dsmem;
  SharedTable* st = reinterpret_cast<SharedTable*>(smem);
  load_shared_table(*st, a.table, pass_slot_width<BW>());
  __syncthreads();

  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + (lane / G);               // scratch slot of this group of lanes
  const int slots_per_cta = NW * a.spw;
  const uint32_t scratch_off = (uint32_t)(a.scratch_off + gid * Scratch<G, BW>::kStreamFloats * 4);
  float* kpbuf = reinterpret_cast<float*>(smem + scratch_off) + Scratch<G, BW>::kFloats;  // 63 floats: current keypoints
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
    solve_stream<G, BW, true>(sv, a.io, a.dm, a.prm, a.S, a.steps, s, works && s < a.S, owner && s < a.S, kpbuf, use_filter,
                              tape.qpos, tape.projected);
  }
}

// dexr_solve_sequences_packed: dexr_sequences_kernel's launch shape and stream slots, stream s with its frames at
// pk.offsets (solve_packed_stream); REC records the tape.  a.steps is not read.
template <int G, int BW, int NW, bool REC>
__global__ void __launch_bounds__(NW * 32, 1) dexr_packed_sequences_kernel(const SeqArgs a, const PackedLayout pk,
                                                                           const dexr_sequences_tape_t tape) {
  unsigned char* const smem = dsmem;
  SharedTable* st = reinterpret_cast<SharedTable*>(smem);
  load_shared_table(*st, a.table, pass_slot_width<BW>());
  __syncthreads();

  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + (lane / G);
  const int slots_per_cta = NW * a.spw;
  const uint32_t scratch_off = (uint32_t)(a.scratch_off + gid * Scratch<G, BW>::kStreamFloats * 4);
  float* kpbuf = reinterpret_cast<float*>(smem + scratch_off) + Scratch<G, BW>::kFloats;
  const int slot = a.spw == GPW ? gid : warp;
  const bool first = (lane / G) == 0;
  const bool owner = a.spw == GPW || first;
  const bool works = owner || a.duo;
  Solver<G, BW> sv;
  sv.init(a.table, a.dm, scratch_off, a.prm, lane);
  if (G == 16 && a.duo) sv.duo = lane / G;
  const bool use_filter = a.prm.lp_alpha >= 0.f && a.prm.lp_alpha <= 1.f;

  for (long long base = 0; base < a.S; base += (long long)gridDim.x * slots_per_cta) {
    const PackedStream ps = packed_stream(pk, base + (long long)slot * gridDim.x + blockIdx.x);
    solve_packed_stream<G, BW, REC>(sv, a.io, a.dm, a.prm, ps, works, owner, kpbuf, use_filter, tape.qpos, tape.projected);
  }
}

// ------------------------------------------------------------------------------------------------
// objective evaluation: one frame per group of G lanes, groups striding over the batch
// ------------------------------------------------------------------------------------------------
// One pass over ~0.5 KB per frame with no iteration: inputs are read with plain loads where they lie (no TMA ring), and the
// table is loaded into shared memory once per CTA.
constexpr int kEvalWarps = 8;

struct EvalArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_eval_t io;
  long long B;
  int in_row;  // floats per frame of the kp/ref input (63 or 3m)
  Dims dm;
  int scratch_off;
};

// (a minimum of 2 CTAs per SM: with none, ptxas gives the 32-lane kernel 64 registers and 8 bytes of spills; now 69-71 and none)
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, 2) dexr_eval_kernel(const EvalArgs a) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);  // (the residual-pass schedule is not read)
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + (warp * GPW + lane / G) * eval_scratch_floats<G>() * 4), a.prm, lane);
  const bool by_kp = a.io.keypoints != nullptr;
  const long long step = (long long)gridDim.x * kEvalWarps * GPW;
  for (long long base = ((long long)blockIdx.x * kEvalWarps + warp) * GPW; base < a.B; base += step) {
    const long long idx = base + lane / G;
    const bool active = idx < a.B;
    const long long f = active ? idx : base;
    FrameInputs in;
    in.kp = by_kp ? a.io.keypoints + f * a.in_row : nullptr;
    in.ref = by_kp ? nullptr : a.io.ref_value + f * a.in_row;
    in.fixed = a.dm.n_fixed > 0 ? a.io.fixed_qpos + f * a.dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = a.io.projected ? a.io.projected + f * a.dm.len_proj : nullptr;
    evaluate_frame(sv, in, a.io, a.dm, f, active);
  }
}

// ------------------------------------------------------------------------------------------------
// backpropagation through the solve: the evaluation kernel's launch shape, one frame per group of G lanes
// ------------------------------------------------------------------------------------------------
struct VjpArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_vjp_t io;
  long long B;
  int in_row;  // floats per frame of the kp/ref input (63 or 3m)
  Dims dm;
  int scratch_off;
};

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, 2) dexr_vjp_kernel(const VjpArgs a) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);  // (the residual-pass schedule is not read)
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + (warp * GPW + lane / G) * VjpScratch<G>::kFloats * 4), a.prm, lane);
  const bool by_kp = a.io.keypoints != nullptr;
  const long long step = (long long)gridDim.x * kEvalWarps * GPW;
  for (long long base = ((long long)blockIdx.x * kEvalWarps + warp) * GPW; base < a.B; base += step) {
    const long long idx = base + lane / G;
    const bool active = idx < a.B;
    const long long f = active ? idx : base;
    FrameInputs in;
    in.kp = by_kp ? a.io.keypoints + f * a.in_row : nullptr;
    in.ref = by_kp ? nullptr : a.io.ref_value + f * a.in_row;
    in.fixed = a.dm.n_fixed > 0 ? a.io.fixed_qpos + f * a.dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = nullptr;  // (vjp_frame reads the flags into its scratch)
    vjp_frame(sv, in, a.io, a.dm, f, active);
  }
}

// ------------------------------------------------------------------------------------------------
// per-frame Jacobians of the solve: the VJP kernel's launch shape, one frame per group of G lanes, one tail per free variable
// ------------------------------------------------------------------------------------------------
struct JacobianArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_jacobian_t io;
  long long B;
  int in_row;  // floats per frame of the kp/ref input (63 or 3m)
  Dims dm;
  int scratch_off;
};

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, 2) dexr_jacobian_kernel(const JacobianArgs a) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);  // (the residual-pass schedule is not read)
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + (warp * GPW + lane / G) * VjpScratch<G>::kFloats * 4), a.prm, lane);
  const bool by_kp = a.io.keypoints != nullptr;
  const long long step = (long long)gridDim.x * kEvalWarps * GPW;
  for (long long base = ((long long)blockIdx.x * kEvalWarps + warp) * GPW; base < a.B; base += step) {
    const long long idx = base + lane / G;
    const bool active = idx < a.B;
    const long long f = active ? idx : base;
    FrameInputs in;
    in.kp = by_kp ? a.io.keypoints + f * a.in_row : nullptr;
    in.ref = by_kp ? nullptr : a.io.ref_value + f * a.in_row;
    in.fixed = a.dm.n_fixed > 0 ? a.io.fixed_qpos + f * a.dm.n_fixed : nullptr;
    in.last = nullptr;
    in.projected = nullptr;  // (jacobian_frame reads the flags into its scratch)
    jacobian_frame(sv, in, a.io, a.dm, f, active);
  }
}

// ------------------------------------------------------------------------------------------------
// backpropagation through the sequence solve: one stream per group of G lanes, walked from its last frame to its first
// ------------------------------------------------------------------------------------------------
struct SeqVjpArgs {
  const dexr_table_t* table;
  dexr_params_t prm;
  dexr_sequences_vjp_t io;
  long long S;
  int steps;
  Dims dm;
  int scratch_off;
  int spw;  // streams per warp: 32 / G, or 1 (the second group of a 16-lane warp walks stream S - 1 and writes nothing)
};

// (32 lanes: a minimum of 2 CTAs per SM caps the kernel at 128 registers, and ptxas spills 4 bytes there)
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_seq_vjp_kernel(const SeqVjpArgs a) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);  // (the residual-pass schedule is not read)
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  const int slot = a.spw == GPW ? gid : warp;
  const bool owner = a.spw == GPW || lane < G;
  const bool use_filter = a.prm.lp_alpha >= 0.f && a.prm.lp_alpha <= 1.f;
  // streams dealt round-robin over the CTAs, as in dexr_sequences_kernel.  A warp whose first group has no stream skips the
  // round (warp-uniform: its other group's stream number is larger) instead of walking stream S - 1 for nothing and taking
  // issue slots from the warps that have one.
  const int first_slot = a.spw == GPW ? warp * GPW : warp;
  for (long long base = 0; base < a.S; base += (long long)gridDim.x * kEvalWarps * a.spw) {
    if (base + (long long)first_slot * gridDim.x + blockIdx.x >= a.S) continue;
    const long long s = base + (long long)slot * gridDim.x + blockIdx.x;
    vjp_stream(sv, a.io, a.dm, a.S, a.steps, s, owner && s < a.S, use_filter);
  }
}

// dexr_solve_sequences_packed_vjp: dexr_seq_vjp_kernel's launch shape and stream slots over the packed streams
// (vjp_packed_stream; a warp without a stream has no steps and moves on).  a.steps is not read.
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_packed_seq_vjp_kernel(const SeqVjpArgs a,
                                                                                               const PackedLayout pk) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  const int slot = a.spw == GPW ? gid : warp;
  const bool owner = a.spw == GPW || lane < G;
  const bool use_filter = a.prm.lp_alpha >= 0.f && a.prm.lp_alpha <= 1.f;
  for (long long base = 0; base < a.S; base += (long long)gridDim.x * kEvalWarps * a.spw) {
    const PackedStream ps = packed_stream(pk, base + (long long)slot * gridDim.x + blockIdx.x);
    vjp_packed_stream(sv, a.io, a.dm, ps, owner, use_filter);
  }
}

// ------------------------------------------------------------------------------------------------
// offline smoothing of packed streams: the packed sequence VJP's launch shape and stream slots, one stream per group of G lanes
// ------------------------------------------------------------------------------------------------
struct SmoothArgs {
  const dexr_table_t* table;
  dexr_params_t prm;  // norm_delta holds the smoothing weight w
  dexr_smooth_t io;
  long long S;
  Dims dm;
  int scratch_off;
};

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_smooth_kernel(const SmoothArgs a, const PackedLayout pk) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  float* const ws = static_cast<float*>(a.io.workspace);
  // one stream per warp: a 16-lane warp's second group idles (measured no slower than two streams per warp, whose outer
  // iteration counts differ, and 1.75x faster on Allegro clips; DESIGN.md 3.12)
  for (long long base = 0; base < a.S; base += (long long)gridDim.x * kEvalWarps) {
    const PackedStream ps = packed_stream(pk, base + (long long)warp * gridDim.x + blockIdx.x);
    smooth_packed_stream(sv, a.io, a.dm, a.prm, ps, lane < G, ws);
  }
}

// backpropagation through the smoother: dexr_smooth_kernel's launch shape, stream slots and workspace
struct SmoothVjpArgs {
  const dexr_table_t* table;
  dexr_params_t prm;  // norm_delta holds the smoothing weight w
  dexr_smooth_vjp_t io;
  long long S;
  Dims dm;
  int scratch_off;
};

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_smooth_vjp_kernel(const SmoothVjpArgs a,
                                                                                           const PackedLayout pk) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  // (one 64-bit stream index live across the stream, not a base and an offset: the 16-lane kernel has 128 registers)
  for (long long i = (long long)warp * gridDim.x + blockIdx.x; i < a.S; i += (long long)gridDim.x * kEvalWarps)
    smooth_vjp_packed_stream(sv, a.io, a.dm, pk, i, lane < G);
}

// the acceleration-penalised smoother and its backpropagation: dexr_smooth_kernel's and dexr_smooth_vjp_kernel's launch
// shapes and stream slots, running smooth_packed_stream<G, true> and smooth_vjp_packed_stream<G, true> (their own kernels, so
// the velocity-only ones keep their code); a.io.smooth_weight holds the acceleration weight c
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_smooth_accel_kernel(const SmoothArgs a,
                                                                                             const PackedLayout pk) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  float* const ws = static_cast<float*>(a.io.workspace);
  for (long long base = 0; base < a.S; base += (long long)gridDim.x * kEvalWarps) {
    const PackedStream ps = packed_stream(pk, base + (long long)warp * gridDim.x + blockIdx.x);
    smooth_packed_stream<G, true>(sv, a.io, a.dm, a.prm, ps, lane < G, ws);
  }
}

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_smooth_accel_vjp_kernel(const SmoothVjpArgs a,
                                                                                                 const PackedLayout pk) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  for (long long i = (long long)warp * gridDim.x + blockIdx.x; i < a.S; i += (long long)gridDim.x * kEvalWarps)
    smooth_vjp_packed_stream<G, true>(sv, a.io, a.dm, pk, i, lane < G);
}

// fixed-lag smoothing of live streams: dexr_smooth_kernel's launch shape and stream slots, K ticks of one stream per warp
// (fixed_lag_tick; a 16-lane warp's second group idles)
struct FixedLagArgs {
  const dexr_table_t* table;
  dexr_params_t prm;  // norm_delta holds the smoothing weight w
  dexr_fixed_lag_t io;
  int32_t* wstatus;  // the status words of the workspace (after the smoother's S (L+1) frames)
  long long S;
  int K;
  int flush;
  Dims dm;
  int scratch_off;
  int pos_off;  // shared memory: each warp's loop state, 2 long longs
};

// The body of dexr_fixed_lag_kernel, dexr_fixed_lag_tape_kernel and dexr_fixed_lag_accel_kernel; REC
// (dexr_fixed_lag_step_tape): fixed_lag_tick's recording into `tape`; ACC (dexr_fixed_lag_step_accel): the ticks and the
// flush of acceleration-penalised streams with the pre-anchor state `acc`.
template <int G, bool REC, bool ACC = false>
__device__ __forceinline__ void fixed_lag_kernel_body(const FixedLagArgs& a, const dexr_fixed_lag_tape_t& tape,
                                                      const dexr_fixed_lag_accel_t* acc = nullptr) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  // the streams dealt as dexr_smooth_kernel deals them.  One loop over (stream, tick) pairs, one tick per iteration: a tick
  // loop nested in the stream loop holds the smoother's loop invariants in registers through every tick.  The loop state
  // (stream, tick) lives in shared memory, read by fixed_lag_tick where it needs it, so that none of it is held in a
  // register across the window solve (the 16-lane kernel spills otherwise).
  volatile long long* const pos = reinterpret_cast<volatile long long*>(dsmem + a.pos_off) + 2 * warp;
  const long long first = (long long)warp * gridDim.x + blockIdx.x;
  if (a.K > 0) {
    if (lane == 0) {
      pos[0] = first;
      pos[1] = 0;
    }
    __syncwarp();
    while (pos[0] < a.S) {
      fixed_lag_tick<G, REC, ACC>(sv, a.io, a.dm, a.prm, a.wstatus, a.K, pos, lane < G, tape.qpos, tape.projected, acc);
      if (lane == 0) {
        if (pos[1] + 1 < a.K) {
          pos[1] = pos[1] + 1;
        } else {
          pos[1] = 0;
          pos[0] = pos[0] + (long long)gridDim.x * kEvalWarps;
        }
      }
      __syncwarp();
    }
  }
  if (a.flush)
    for (long long s = first; s < a.S; s += (long long)gridDim.x * kEvalWarps)
      fixed_lag_flush<G, ACC>(sv, a.io, a.dm, a.prm, s, lane < G, acc);
}

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_kernel(const FixedLagArgs a) {
  fixed_lag_kernel_body<G, false>(a, dexr_fixed_lag_tape_t{nullptr, nullptr});
}

// dexr_fixed_lag_step_tape: dexr_fixed_lag_kernel with fixed_lag_tick's recording switched on.
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_tape_kernel(const FixedLagArgs a,
                                                                                               const dexr_fixed_lag_tape_t tape) {
  fixed_lag_kernel_body<G, true>(a, tape);
}

// dexr_fixed_lag_step_accel: dexr_fixed_lag_kernel with the acceleration-penalised window solve and the pre-anchor state
// (its own kernel, so that the velocity-only one keeps its code; the smoother's workspace per frame is SmoothAccWs<G>).
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_accel_kernel(
    const FixedLagArgs a, const __grid_constant__ dexr_fixed_lag_accel_t acc) {
  fixed_lag_kernel_body<G, false, true>(a, dexr_fixed_lag_tape_t{nullptr, nullptr}, &acc);
}

// dexr_fixed_lag_step_accel_tape: dexr_fixed_lag_accel_kernel with fixed_lag_tick's recording switched on.
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_accel_tape_kernel(
    const FixedLagArgs a, const dexr_fixed_lag_tape_t tape, const __grid_constant__ dexr_fixed_lag_accel_t acc) {
  fixed_lag_kernel_body<G, true, true>(a, tape, &acc);
}

// backpropagation through fixed-lag smoothing: dexr_smooth_vjp_kernel's launch shape, the streams dealt as
// dexr_fixed_lag_kernel deals them, a stream's ticks walked in reverse on its warp (a 16-lane warp's second group idles)
struct FixedLagVjpArgs {
  const dexr_table_t* table;
  dexr_params_t prm;  // norm_delta holds the smoothing weight w
  dexr_fixed_lag_vjp_t io;
  dexr_smooth_vjp_t wio;  // the window VJP's view of the workspace (fixed_lag_vjp_window_io)
  PackedLayout wpk;       // its packed layout: stream s's window is packed stream 2 s
  FixedLagVjpWs ws;
  long long S;
  int K;
  Dims dm;
  int scratch_off;
  int pos_off;  // shared memory: each warp's loop state, 2 long longs
};

// The body of dexr_fixed_lag_vjp_kernel and dexr_fixed_lag_accel_vjp_kernel; ACC (dexr_fixed_lag_step_accel_vjp): the
// accelerated window VJP (smooth_vjp_packed_stream<G, true, true>, the window view's c and H_k flags set by the launch) and
// the fixed_lag_vjp_* helpers' pre-anchor rows and C2, with `acc` and the workspace's `pw`.
template <int G, bool ACC = false>
__device__ __forceinline__ void fixed_lag_vjp_kernel_body(const FixedLagVjpArgs& a, const dexr_fixed_lag_accel_vjp_t* acc = nullptr,
                                                          const FixedLagPreWs* pw = nullptr) {
  load_shared_table(*reinterpret_cast<SharedTable*>(dsmem), a.table);
  __syncthreads();
  constexpr int GPW = 32 / G;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int gid = warp * GPW + lane / G;
  Solver<G, 0> sv;
  sv.init(a.table, a.dm, (uint32_t)(a.scratch_off + gid * VjpScratch<G>::kFloats * 4), a.prm, lane);
  // One loop over (stream, tick) pairs, the ticks of a stream from K-1 down to 0, one per iteration; the loop state lives in
  // shared memory as in dexr_fixed_lag_kernel, so that none of it is held in a register across the window VJP.  Its address
  // is recomputed at each use (`pos()`), and the lane read again from threadIdx: held through the window VJP, either is a
  // register the 16-lane kernel does not have (it spills otherwise).
  auto pos = [&]() {
    return reinterpret_cast<volatile long long*>(dsmem + a.pos_off) + 2 * opaque((uint32_t)(threadIdx.x >> 5));
  };
  const long long first = (long long)warp * gridDim.x + blockIdx.x;
  if (a.K == 0) {
    for (long long s = first; s < a.S; s += (long long)gridDim.x * kEvalWarps)
      fixed_lag_vjp_begin<G, ACC>(sv, a.io, a.ws, a.dm, s, 0, (threadIdx.x & 31) < G, acc, pw);
    return;
  }
  if ((threadIdx.x & 31) == 0) {
    pos()[0] = first;
    pos()[1] = a.K - 1;
  }
  __syncwarp();
  while (pos()[0] < a.S) {
    if (pos()[1] == a.K - 1) fixed_lag_vjp_begin<G, ACC>(sv, a.io, a.ws, a.dm, pos()[0], a.K, (threadIdx.x & 31) < G, acc, pw);
    if (fixed_lag_vjp_rebuild<G, ACC>(sv, a.io, a.ws, a.dm, a.K, pos(), (threadIdx.x & 31) < G, acc, pw)) {
      smooth_vjp_packed_stream<G, ACC, ACC>(sv, a.wio, a.dm, a.wpk, 2 * pos()[0], (threadIdx.x & 31) < G);
      fixed_lag_vjp_scatter<G, ACC>(sv, a.io, a.ws, a.dm, a.K, pos(), (threadIdx.x & 31) < G, acc, pw);
    }
    if ((threadIdx.x & 31) == 0) {
      volatile long long* const p = pos();
      if (p[1] > 0) {
        p[1] = p[1] - 1;
      } else {
        p[1] = a.K - 1;
        p[0] = p[0] + (long long)gridDim.x * kEvalWarps;
      }
    }
    __syncwarp();
  }
}

template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_vjp_kernel(const FixedLagVjpArgs a) {
  fixed_lag_vjp_kernel_body<G>(a);
}

// dexr_fixed_lag_step_accel_vjp: dexr_fixed_lag_vjp_kernel through acceleration-penalised windows (its own kernel, so that
// the velocity-only one keeps its code; a.ws.smooth holds SmoothAccWs<G> per frame, `pw` the pre-anchor flags and C2).
template <int G>
__global__ void __launch_bounds__(kEvalWarps * 32, G == 16 ? 2 : 1) dexr_fixed_lag_accel_vjp_kernel(
    const FixedLagVjpArgs a, const __grid_constant__ dexr_fixed_lag_accel_vjp_t acc, const __grid_constant__ FixedLagPreWs pw) {
  fixed_lag_vjp_kernel_body<G, true>(a, &acc, &pw);
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

constexpr int kQueueSlots = 16;

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
  int smem_optin = 0;  // dynamic shared memory a CTA may opt in to
  // Tile queues of the frames kernel: kQueueSlots zeroed slots, each with the event recorded behind the last launch that
  // used it.  A launch takes a slot whose event has completed: that launch has ended, and its last CTA left the slot
  // zeroed.  So two launches that can overlap (two streams, or this robot in two groups of one mixed call) never share a
  // slot, with no memset or extra kernel per call.  When every slot is in use, the launch waits on its stream for the
  // next slot's event (work enqueued earlier: this cannot deadlock).  queue_mu covers the choice and the launch.
  QueueSlot* queue_dev = nullptr;
  cudaEvent_t queue_ev[kQueueSlots] = {};
  int queue_next = 0;
  std::mutex queue_mu;
};

static int frames_max_tile(int lanes) { return lanes == 16 ? 64 : 32; }  // frames per ring stage (shared memory budget)

// Input ring depth of the frames kernel: 4 stages (measured: DESIGN.md 3.1); DEXR_FRAMES_STAGES=2|3|4 (read per call)
// overrides for A/B runs.  fill_frame_args takes fewer where a CTA's shared memory would not fit.
static int frames_stages() {
  const char* e = getenv("DEXR_FRAMES_STAGES");
  const int s = e ? atoi(e) : 0;
  return s >= 2 && s <= 4 ? s : 4;
}

// DEXR_FRAMES_QUEUE=0 (read per call) hands the tiles out by static striding instead of the grid-wide queue, for A/B runs.
static bool frames_queue_enabled() {
  const char* e = getenv("DEXR_FRAMES_QUEUE");
  return !(e && atoi(e) == 0);
}
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
  r->smem_optin = (int)prop.sharedMemPerBlockOptin;
  // the frames kernel's tile queue slots start zeroed (the synchronise: before any launch on any stream can read them)
  ce = cudaMalloc(&r->queue_dev, kQueueSlots * sizeof(QueueSlot));
  if (ce == cudaSuccess) ce = cudaMemset(r->queue_dev, 0, kQueueSlots * sizeof(QueueSlot));
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  for (int i = 0; i < kQueueSlots && ce == cudaSuccess; ++i) ce = cudaEventCreateWithFlags(&r->queue_ev[i], cudaEventDisableTiming);
  if (ce != cudaSuccess) {
    dexr_robot_destroy(r);
    return fail(DEXR_E_CUDA, "allocating the frames kernel's tile queues failed: %s", cudaGetErrorString(ce));
  }
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
size_t dexr_eval_sizeof(void) { return sizeof(dexr_eval_t); }
size_t dexr_vjp_sizeof(void) { return sizeof(dexr_vjp_t); }
size_t dexr_sequences_tape_sizeof(void) { return sizeof(dexr_sequences_tape_t); }
size_t dexr_sequences_vjp_sizeof(void) { return sizeof(dexr_sequences_vjp_t); }
size_t dexr_jacobian_sizeof(void) { return sizeof(dexr_jacobian_t); }

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
  for (int i = 0; i < kQueueSlots; ++i)
    if (robot->queue_ev[i]) cudaEventDestroy(robot->queue_ev[i]);
  if (robot->queue_dev) cudaFree(robot->queue_dev);
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
template <int G, int BW, int NCW>
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
  // Ring depth: frames_stages() (4), fewer where the shared memory of the CTA would not fit.  Per stage: the tile, two
  // barriers and the tile's first frame (8 bytes each), its frame claim counter and its size (4 bytes each).
  constexpr int GPW = 32 / G;
  const int scratch_bytes = NCW * GPW * Scratch<G, BW>::kFloats * 4;
  int S = frames_stages();
  auto layout = [&](int s) {
    a.stages = s;
    a.bar_off = a.ring_off + s * a.stage_bytes;
    a.scratch_off = round_up(a.bar_off + s * 32, 16);
    return a.scratch_off + scratch_bytes;
  };
  while (S > 2 && layout(S) > r->smem_optin) --S;
  const int smem = layout(S);
  // the queue's smallest tile: about two rounds of the CTA's warps over the ring's stages (block 16, 24 warps, 4 stages:
  // 24 frames).  Every tile costs a claim and a staging, and with smaller tiles the warps wait for stages at the end of
  // the launch more than the finer split saves (DESIGN.md 3.1).  Tiles that are not a multiple of 4 (exact one-round
  // tiles) never shrink.
  a.min_chunk = (T & 3) ? T : std::min(T, round_up((2 * kRound + S - 1) / S, 4));
  return smem;
}

// The queue's schedule (frames_group): after the grid's first tiles, full tiles while more than stages x grid x (the next
// size) frames would be left, then tiles of half the size, and so on down to min_chunk.  Sizes are multiples of 4, so
// every tile's inputs stay 16-byte aligned for the bulk copy; only the batch's ragged end is smaller.  A CTA holds at
// most `stages` claimed tiles, so near the end what it holds is at most its share of the rest, and the CTAs end within
// about one smallest tile of each other: guided self-scheduling, with the sizes fixed per launch.
static void plan_queue(FrameArgs& a, int grid) {
  long long rest = a.B - (long long)grid * a.T;
  const long long share = (long long)a.stages * grid;
  int c = a.T;
  a.n_levels = 0;
  while (rest > 0) {
    const int nc = std::max(a.min_chunk, round_up(c / 2, 4));
    const bool last = c <= a.min_chunk || a.n_levels == kMaxLevels - 1;
    const long long n = last ? (rest + c - 1) / c : std::max(0LL, (rest - share * nc) / c);
    a.lv_size[a.n_levels] = c;
    a.lv_tiles[a.n_levels] = (int)n;
    ++a.n_levels;
    rest -= n * c;
    c = nc;
  }
}

// DEXR_FRAMES_PDL=0 (read per call) launches the single-robot frames kernel without programmatic dependent launch, for
// A/B runs.
static bool frames_pdl_enabled() {
  const char* e = getenv("DEXR_FRAMES_PDL");
  return !(e && atoi(e) == 0);
}

// The single-robot frames kernel, launched with programmatic stream serialisation (see grid_dep_launch).
template <class K>
static cudaError_t launch_frames_kernel(K kern, int grid, int block, int smem, cudaStream_t stream, const FrameArgs& a) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = frames_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, a);
}

template <int G, int BW, int NCW>
static int launch_frames(dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, cudaStream_t stream, int slots, int tile) {
  FrameArgs a;
  if (slots <= 0) slots = r->num_sms;  // one persistent CTA per SM; a mixed launch passes its own CTA count and tile size
  const int smem = fill_frame_args<G, BW, NCW>(r, prm, io, B, slots, a, tile);
  auto kern = dexr_frames_kernel<G, BW, NCW>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = std::min(a.ntiles, slots);
#ifdef DEXR_EXP_TIMELINE
  a.timeline = g_timeline;
#endif
  if ((long long)grid * a.T >= B || !frames_queue_enabled()) {  // every CTA's first tile covers the batch: no queue
    CUDA_TRY(launch_frames_kernel(kern, grid, (NCW + 1) * 32, smem, stream, a));
  } else {
    std::lock_guard<std::mutex> lk(r->queue_mu);
    int slot = -1;
    for (int k = 0; k < kQueueSlots && slot < 0; ++k) {
      const int i = (r->queue_next + k) % kQueueSlots;
      const cudaError_t q = cudaEventQuery(r->queue_ev[i]);
      if (q == cudaSuccess) slot = i;
      else if (q == cudaErrorNotReady) cudaGetLastError();  // (not an error: the slot is in use)
      else return fail(DEXR_E_CUDA, "cudaEventQuery on a tile queue slot failed: %s", cudaGetErrorString(q));
    }
    if (slot < 0) {
      slot = r->queue_next;
      CUDA_TRY(cudaStreamWaitEvent(stream, r->queue_ev[slot], 0));
    }
    r->queue_next = (slot + 1) % kQueueSlots;
    a.queue = r->queue_dev + slot;
    plan_queue(a, grid);
    CUDA_TRY(launch_frames_kernel(kern, grid, (NCW + 1) * 32, smem, stream, a));
    CUDA_TRY(cudaEventRecord(r->queue_ev[slot], stream));
  }
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, (NCW + 1) * 32, smem, a.T, G, NCW, r->last.kernels_launched + 1};
  }
  return 0;
}

// Consumer warps per CTA for each solver kind (index = solver_kind()), counted with the producer.  One CTA per SM; ptxas splits
// the 64 K x 32-bit register file over the SM's four sub-partitions (16 K registers each, warps dealt round-robin), so the
// caps are 168 registers per thread at 12 warps, 128 at 13-16, 96 at 17-20, 80 at 21-24 and 72 at 25-28: a count between
// two steps buys no registers.  Measured on H100 SXM (400 W, 65 536 frames per launch, 16 | 14 | 12 warps, ms): every dense
// and arrow kind is fastest with 16 warps despite the spills at 128 registers -- LEAP DexPilot (dense 16) 1.77 | 1.86 | 1.80,
// Ability (dense 16, mimic) 1.52 | 1.67 | 1.75, Shadow position (arrow) 3.21 | 3.37 | 3.45, SVH (dense 32) 4.34 | 4.75 | 4.80.
// The block-diagonal solver needs 119 registers and runs fastest with 24 warps at 80 (sweep: DESIGN.md 3.1).
// DEXR_FRAMES_WARPS="a,b,c,d" overrides for A/B runs: block 16 | 20 | 24 | 28, the other kinds 16 | 14 | 12.
static const int* frames_warps() {
  static int w[4] = {24, 16, 16, 16};
  static const bool init = [] {
    if (const char* e = getenv("DEXR_FRAMES_WARPS")) {
      int v[4];
      if (sscanf(e, "%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3]) == 4) {
        if (v[0] == 16 || v[0] == 20 || v[0] == 24 || v[0] == 28) w[0] = v[0];
        for (int i = 1; i < 4; ++i)
          if (v[i] == 16 || v[i] == 14 || v[i] == 12) w[i] = v[i];
      }
    }
    return true;
  }();
  (void)init;
  return w;
}

template <int G, int BW>
static int launch_frames_warps(int warps, dexr_robot* r, const dexr_params_t* prm, const dexr_frames_t* io, long long B, cudaStream_t stream, int slots, int tile) {
  if constexpr (BW > 0) {
    if (warps == 20) return launch_frames<G, BW, 19>(r, prm, io, B, stream, slots, tile);
    if (warps == 24) return launch_frames<G, BW, 23>(r, prm, io, B, stream, slots, tile);
    if (warps == 28) return launch_frames<G, BW, 27>(r, prm, io, B, stream, slots, tile);
  } else {
    if (warps == 12) return launch_frames<G, BW, 11>(r, prm, io, B, stream, slots, tile);
    if (warps == 14) return launch_frames<G, BW, 13>(r, prm, io, B, stream, slots, tile);
  }
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

static int check_eval_io(const dexr_table_t& t, const dexr_eval_t* io, const dexr_params_t* prm) {
  if (const char* msg = eval_io_error(t, *io, *prm)) return fail(DEXR_E_INVALID, "%s", msg);
  return 0;
}

// The loss fields of check_params: an evaluation ignores the solver's.
static int check_loss_params(const dexr_params_t* p) {
  if (!(p->huber_delta > 0.f)) return fail(DEXR_E_INVALID, "huber_delta must be > 0");
  if (!(p->norm_delta >= 0.f)) return fail(DEXR_E_INVALID, "norm_delta must be >= 0");
  if (p->preprocess < 0 || p->preprocess > 2) return fail(DEXR_E_INVALID, "preprocess must be 0 (none), 1 (right hand) or 2 (left hand)");
  return 0;
}

// CTAs per SM of the evaluation kernel: as many as are resident at once (registers and shared memory allow), one wave that
// grid-strides over the batch.  DEXR_EVAL_CTAS_PER_SM (read per call) caps it for A/B runs.  The choice is measured in
// DESIGN.md section 3 ("Objective evaluation").
// The VJP and Jacobian kernels use the same rule and cap.
template <class K>
static int eval_ctas_per_sm(K kern, int smem, int* out) {
  int resident = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, kEvalWarps * 32, smem));
  int n = std::max(1, resident);
  if (const char* e = getenv("DEXR_EVAL_CTAS_PER_SM"))
    if (atoi(e) > 0) n = std::min(n, atoi(e));
  *out = n;
  return 0;
}

template <int G>
static int launch_eval(dexr_robot* r, const dexr_params_t* prm, const dexr_eval_t* io, long long B, cudaStream_t stream) {
  const dexr_table_t& t = r->host;
  EvalArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  a.io = *io;
  a.B = B;
  a.in_row = io->keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * t.n_res;
  a.dm = make_dims(t);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * eval_scratch_floats<G>() * 4;  // below the 48 KB default
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(dexr_eval_kernel<G>, smem, &per_sm)) return e;
  const long long ctas = (B + kEvalWarps * GPW - 1) / (kEvalWarps * GPW);
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  dexr_eval_kernel<G><<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_eval_objective(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_eval_t* io,
                                   int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_eval_objective: null argument");
  if (num_frames < 0) return fail(DEXR_E_INVALID, "num_frames < 0");
  if (int e = check_eval_io(robot->host, io, params)) return e;
  if (int e = check_loss_params(params)) return e;
  if (num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_eval<16>(r, params, io, num_frames, stream)
                                   : launch_eval<32>(r, params, io, num_frames, stream);
}

static int check_vjp_io(const dexr_table_t& t, const dexr_vjp_t* io, const dexr_params_t* prm) {
  if (const char* msg = vjp_io_error(t, *io, *prm)) return fail(DEXR_E_INVALID, "%s", msg);
  return 0;
}

template <int G>
static int launch_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_vjp_t* io, long long B, cudaStream_t stream) {
  const dexr_table_t& t = r->host;
  VjpArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  a.io = *io;
  a.B = B;
  a.in_row = io->keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * t.n_res;
  a.dm = make_dims(t);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;  // 16 lanes: 77 KB, 32 lanes: 101 KB
  auto kern = dexr_vjp_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const long long ctas = (B + kEvalWarps * GPW - 1) / (kEvalWarps * GPW);
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_solve_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_vjp_t* io,
                              int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_vjp: null argument");
  if (num_frames < 0) return fail(DEXR_E_INVALID, "num_frames < 0");
  if (int e = check_vjp_io(robot->host, io, params)) return e;
  if (int e = check_loss_params(params)) return e;
  if (num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_vjp<16>(r, params, io, num_frames, stream)
                                   : launch_vjp<32>(r, params, io, num_frames, stream);
}

template <int G>
static int launch_jacobian(dexr_robot* r, const dexr_params_t* prm, const dexr_jacobian_t* io, long long B,
                           cudaStream_t stream) {
  const dexr_table_t& t = r->host;
  JacobianArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  a.io = *io;
  a.B = B;
  a.in_row = io->keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * t.n_res;
  a.dm = make_dims(t);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;  // as the VJP kernel's
  auto kern = dexr_jacobian_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const long long ctas = (B + kEvalWarps * GPW - 1) / (kEvalWarps * GPW);
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_solve_jacobian(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_jacobian_t* io,
                                   int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_jacobian: null argument");
  if (num_frames < 0) return fail(DEXR_E_INVALID, "num_frames < 0");
  if (const char* msg = jacobian_io_error(robot->host, *io, *params)) return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_jacobian<16>(r, params, io, num_frames, stream)
                                   : launch_jacobian<32>(r, params, io, num_frames, stream);
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
    const int need = with_solver(k, [&](auto s) {
      return fill_frame_args<decltype(s)::G, decltype(s)::BW, NCW>(r, g.params, &g.io, g.num_frames, sms, a);
    });
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

#ifdef DEXR_EXP_TIMELINE
// Experiment builds only: the device buffer the frames kernel records its events into from the next launch on (nullptr:
// none).  Returns the buffer's size in bytes (layout: Timeline).
extern "C" int64_t dexr_exp_timeline(void* buffer) {
  g_timeline = static_cast<unsigned long long*>(buffer);
  return (int64_t)kTlCtas * 32 * (1 + 4 * kTlEvents) * 8;
}
#endif

// Launch shape of the sequences kernels for S streams: sets a.spw and a.duo, returns the grid.
// A stream is serial in time and latency bound, so streams are spread over as many warps and SMs as there are: while one
// warp per stream fits into one wave of CTAs (S <= SMs x warps per CTA), a warp carries ONE stream (the second group of a
// 16-lane solver idles); beyond that two 16-lane streams share a warp.  One CTA per SM, two when streams are plentiful.
template <int G>
static int sequences_shape(const dexr_robot* r, long long S, SeqArgs& a) {
  constexpr int GPW = 32 / G;
  const long long warps_one_wave = (long long)r->num_sms * kSeqNW;
  a.spw = (GPW > 1 && S > warps_one_wave) ? GPW : 1;
  static const int spw_env = [] { const char* e = getenv("DEXR_SEQ_PAIR"); return e ? atoi(e) : -1; }();  // A/B: 1 = always pair
  if (spw_env == 1) a.spw = GPW;
  const char* duo_env = getenv("DEXR_SEQ_DUO");  // 0 = off (read per call: tests compare the two modes in one process)
  a.duo = (G == 16 && a.spw == 1 && !(duo_env && atoi(duo_env) == 0)) ? 1 : 0;
  const long long per_cta = (long long)kSeqNW * a.spw;
  const long long ctas = std::max<long long>(1, (S + a.spw - 1) / a.spw);  // at least one warp's worth of streams per CTA
  return (int)std::min<long long>(ctas, (long long)r->num_sms * (S >= (long long)r->num_sms * per_cta * 2 ? 2 : 1));
}

template <int G, int BW>
static int launch_sequences(dexr_robot* r, const dexr_params_t* prm, const dexr_sequences_t* io, long long S, int steps,
                            cudaStream_t stream, const dexr_sequences_tape_t* tape = nullptr) {
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
  const int smem = a.scratch_off + groups * Scratch<G, BW>::kStreamFloats * 4;
  auto kern = dexr_sequences_kernel<G, BW, kSeqNW>;
  auto kern_tape = dexr_sequences_tape_kernel<G, BW, kSeqNW>;
  if (tape) CUDA_TRY(cudaFuncSetAttribute(kern_tape, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  else CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = sequences_shape<G>(r, S, a);
  if (tape) kern_tape<<<grid, kSeqNW * 32, smem, stream>>>(a, *tape);
  else kern<<<grid, kSeqNW * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kSeqNW * 32, smem, 0, G, kSeqNW, r->last.kernels_launched + 1};
  }
  return 0;
}

// dexr_solve_sequences_packed: launch_sequences for S packed streams (same shape, spw, duo and grid).
template <int G, int BW>
static int launch_packed_sequences(dexr_robot* r, const dexr_params_t* prm, const dexr_sequences_t* io, const PackedLayout& pk,
                                   cudaStream_t stream, const dexr_sequences_tape_t* tape) {
  SeqArgs a{};
  a.table = r->table_dev;
  a.prm = sequence_params(*prm);
  a.io = *io;
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  const int smem = a.scratch_off + kSeqNW * (32 / G) * Scratch<G, BW>::kStreamFloats * 4;
  auto kern = dexr_packed_sequences_kernel<G, BW, kSeqNW, false>;
  auto kern_tape = dexr_packed_sequences_kernel<G, BW, kSeqNW, true>;
  CUDA_TRY(cudaFuncSetAttribute(tape ? kern_tape : kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = sequences_shape<G>(r, pk.S, a);
  if (tape) kern_tape<<<grid, kSeqNW * 32, smem, stream>>>(a, pk, *tape);
  else kern<<<grid, kSeqNW * 32, smem, stream>>>(a, pk, dexr_sequences_tape_t{nullptr, nullptr});
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

extern "C" int dexr_solve_sequences_tape(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                                         const dexr_sequences_tape_t* tape, int64_t num_streams, int64_t num_steps,
                                         void* cuda_stream) {
  if (!robot || !params || !io || !tape) return fail(DEXR_E_INVALID, "dexr_solve_sequences_tape: null argument");
  if (num_streams < 0 || num_steps < 0 || num_steps > INT32_MAX) return fail(DEXR_E_INVALID, "bad sizes");
  if (num_streams == 0 || num_steps == 0) return 0;
  if (int e = check_params(params)) return e;
  if (int e = check_sequences_io(robot->host, io, params)) return e;
  if (!tape->qpos) return fail(DEXR_E_INVALID, "tape->qpos is required");
  if (robot->host.loss == DEXR_LOSS_DEXPILOT && (!tape->projected || !io->projected))
    return fail(DEXR_E_INVALID, "DexPilot: the flag tape needs tape->projected and io->projected");
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const dexr_sequences_tape_t tp{tape->qpos, robot->host.loss == DEXR_LOSS_DEXPILOT ? tape->projected : nullptr};
  return with_solver(solver_kind(r->host, arrow_enabled()), [&](auto s) {
    return launch_sequences<decltype(s)::G, decltype(s)::BW>(r, params, io, num_streams, (int)num_steps, stream, &tp);
  });
}

// Launch shape of the sequence VJP: the VJP kernel's CTA (kEvalWarps warps, as many CTAs per SM as are resident, one wave
// that strides over the streams), one stream per group of G lanes (two per warp for 16-lane robots: 12-14 % faster than
// one on H100, DESIGN.md section 3.9).  DEXR_SEQ_VJP_SPW=1 (read per call) gives every 16-lane stream a warp of its own and
// DEXR_EVAL_CTAS_PER_SM caps the CTAs per SM, for A/B runs.
template <int G>
static int launch_seq_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_sequences_vjp_t* io, long long S, int steps,
                          cudaStream_t stream) {
  const dexr_table_t& t = r->host;
  SeqVjpArgs a{};
  a.table = r->table_dev;
  a.prm = sequence_params(*prm);
  a.io = *io;
  a.S = S;
  a.steps = steps;
  a.dm = make_dims(t);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  a.spw = GPW;
  if (const char* e = getenv("DEXR_SEQ_VJP_SPW"))
    if (atoi(e) == 1) a.spw = 1;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_seq_vjp_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  // a stream is serial in time: deal the streams over as many CTAs as are resident (a warp's worth per CTA at least), so
  // that a few hundred streams still reach every SM; the warps left without a stream skip the round
  const long long ctas = (S + a.spw - 1) / a.spw;
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_solve_sequences_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_vjp_t* io,
                                        int64_t num_streams, int64_t num_steps, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_sequences_vjp: null argument");
  if (num_streams < 0 || num_steps < 0 || num_steps > INT32_MAX) return fail(DEXR_E_INVALID, "bad sizes");
  if (const char* msg = seq_vjp_io_error(robot->host, *io, *params)) return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0 || num_steps == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_seq_vjp<16>(r, params, io, num_streams, (int)num_steps, stream)
                                   : launch_seq_vjp<32>(r, params, io, num_streams, (int)num_steps, stream);
}

extern "C" int dexr_solve_sequences_packed(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                                           const dexr_sequences_tape_t* tape, const int64_t* offsets, int64_t num_streams, int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_sequences_packed: null argument");
  if (const char* msg = packed_io_error(robot->host, *io, tape, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (num_streams == 0 || num_frames == 0) return 0;
  if (int e = check_params(params)) return e;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  dexr_sequences_tape_t tp{nullptr, nullptr};
  if (tape) tp = dexr_sequences_tape_t{tape->qpos, robot->host.loss == DEXR_LOSS_DEXPILOT ? tape->projected : nullptr};
  return with_solver(solver_kind(r->host, arrow_enabled()), [&](auto s) {
    return launch_packed_sequences<decltype(s)::G, decltype(s)::BW>(r, params, io, pk, stream, tape ? &tp : nullptr);
  });
}

// dexr_solve_sequences_packed_vjp: launch_seq_vjp's shape (and A/B switches) for S packed streams.
template <int G>
static int launch_packed_seq_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_sequences_vjp_t* io, const PackedLayout& pk,
                                 cudaStream_t stream) {
  SeqVjpArgs a{};
  a.table = r->table_dev;
  a.prm = sequence_params(*prm);
  a.io = *io;
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  a.spw = GPW;
  if (const char* e = getenv("DEXR_SEQ_VJP_SPW"))
    if (atoi(e) == 1) a.spw = 1;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_packed_seq_vjp_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const long long ctas = (pk.S + a.spw - 1) / a.spw;
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a, pk);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" int dexr_solve_sequences_packed_vjp(const dexr_robot_t* robot, const dexr_params_t* params,
                                               const dexr_sequences_vjp_t* io, const int64_t* offsets, int64_t num_streams, int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_solve_sequences_packed_vjp: null argument");
  if (const char* msg = packed_io_error(robot->host, *io, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0 || num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  return eval_lanes(r->host) == 16 ? launch_packed_seq_vjp<16>(r, params, io, pk, stream)
                                   : launch_packed_seq_vjp<32>(r, params, io, pk, stream);
}

// dexr_smooth_sequences_packed: dexr_packed_seq_vjp_kernel's CTA and occupancy rule, one stream per warp, the smoothing
// weight passed in params.norm_delta.
template <int G>
static int launch_smooth(dexr_robot* r, const dexr_params_t* prm, const dexr_smooth_t* io, const PackedLayout& pk,
                         cudaStream_t stream) {
  SmoothArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_smooth_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const long long ctas = pk.S;
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a, pk);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

// dexr_smooth_sequences_packed_accel: launch_smooth's CTA and occupancy rule.
template <int G>
static int launch_smooth_accel(dexr_robot* r, const dexr_params_t* prm, const dexr_smooth_t* io, float accel,
                               const PackedLayout& pk, cudaStream_t stream) {
  SmoothArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  a.io.smooth_weight = accel;  // (w is in a.prm.norm_delta)
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_smooth_accel_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const int grid = (int)std::min<long long>(pk.S, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a, pk);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" size_t dexr_smooth_sizeof(void) { return sizeof(dexr_smooth_t); }

extern "C" size_t dexr_smooth_workspace_bytes(const dexr_robot_t* robot, int64_t num_frames) {
  return robot ? smooth_workspace_bytes(robot->host, num_frames) : 0;
}

extern "C" int dexr_smooth_sequences_packed(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_smooth_t* io,
                                            const int64_t* offsets, int64_t num_streams, int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_smooth_sequences_packed: null argument");
  if (const char* msg = smooth_io_error(robot->host, *io, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  return eval_lanes(r->host) == 16 ? launch_smooth<16>(r, params, io, pk, stream) : launch_smooth<32>(r, params, io, pk, stream);
}

// dexr_smooth_sequences_packed_vjp: launch_smooth's CTA and occupancy rule.
template <int G>
static int launch_smooth_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_smooth_vjp_t* io, const PackedLayout& pk,
                             cudaStream_t stream) {
  SmoothVjpArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_smooth_vjp_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const long long ctas = pk.S;
  const int grid = (int)std::min<long long>(ctas, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a, pk);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

// dexr_smooth_sequences_packed_accel_vjp: launch_smooth's CTA and occupancy rule.
template <int G>
static int launch_smooth_accel_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_smooth_vjp_t* io, float accel,
                                   const PackedLayout& pk, cudaStream_t stream) {
  SmoothVjpArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  a.io.smooth_weight = accel;  // (w is in a.prm.norm_delta)
  a.S = pk.S;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  const int smem = a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4;
  auto kern = dexr_smooth_accel_vjp_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const int grid = (int)std::min<long long>(pk.S, (long long)r->num_sms * per_sm);
  kern<<<grid, kEvalWarps * 32, smem, stream>>>(a, pk);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" size_t dexr_smooth_vjp_sizeof(void) { return sizeof(dexr_smooth_vjp_t); }

extern "C" int dexr_smooth_sequences_packed_vjp(const dexr_robot_t* robot, const dexr_params_t* params,
                                                const dexr_smooth_vjp_t* io, const int64_t* offsets, int64_t num_streams,
                                                int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_smooth_sequences_packed_vjp: null argument");
  if (const char* msg = smooth_vjp_io_error(robot->host, *io, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0 || num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  return eval_lanes(r->host) == 16 ? launch_smooth_vjp<16>(r, params, io, pk, stream)
                                   : launch_smooth_vjp<32>(r, params, io, pk, stream);
}

extern "C" size_t dexr_smooth_accel_workspace_bytes(const dexr_robot_t* robot, int64_t num_frames) {
  return robot ? smooth_accel_workspace_bytes(robot->host, num_frames) : 0;
}

extern "C" int dexr_smooth_sequences_packed_accel(const dexr_robot_t* robot, const dexr_params_t* params,
                                                  const dexr_smooth_t* io, float accel_weight, const int64_t* offsets,
                                                  int64_t num_streams, int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_smooth_sequences_packed_accel: null argument");
  if (accel_weight == 0.f)
    return dexr_smooth_sequences_packed(robot, params, io, offsets, num_streams, num_frames, cuda_stream);
  if (const char* msg = smooth_io_error(robot->host, *io, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (const char* msg = smooth_accel_error(robot->host, accel_weight, io->workspace, io->workspace_bytes, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  return eval_lanes(r->host) == 16 ? launch_smooth_accel<16>(r, params, io, accel_weight, pk, stream)
                                   : launch_smooth_accel<32>(r, params, io, accel_weight, pk, stream);
}

extern "C" int dexr_smooth_sequences_packed_accel_vjp(const dexr_robot_t* robot, const dexr_params_t* params,
                                                      const dexr_smooth_vjp_t* io, float accel_weight, const int64_t* offsets,
                                                      int64_t num_streams, int64_t num_frames, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_smooth_sequences_packed_accel_vjp: null argument");
  if (accel_weight == 0.f)
    return dexr_smooth_sequences_packed_vjp(robot, params, io, offsets, num_streams, num_frames, cuda_stream);
  if (const char* msg = smooth_vjp_io_error(robot->host, *io, *params, offsets, num_streams, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (const char* msg = smooth_accel_error(robot->host, accel_weight, io->workspace, io->workspace_bytes, num_frames))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0 || num_frames == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const PackedLayout pk{offsets, num_streams, num_frames};
  return eval_lanes(r->host) == 16 ? launch_smooth_accel_vjp<16>(r, params, io, accel_weight, pk, stream)
                                   : launch_smooth_accel_vjp<32>(r, params, io, accel_weight, pk, stream);
}

// dexr_fixed_lag_step: launch_smooth's CTA and occupancy rule.  `tape`: dexr_fixed_lag_step_tape's recording; `acc`:
// dexr_fixed_lag_step_accel's pre-anchor state (dexr_fixed_lag_accel_kernel, its own occupancy, the status words after the
// accel smoother's workspace); both: dexr_fixed_lag_step_accel_tape (dexr_fixed_lag_accel_tape_kernel).
template <int G>
static int launch_fixed_lag(dexr_robot* r, const dexr_params_t* prm, const dexr_fixed_lag_t* io, long long S, int K,
                            cudaStream_t stream, const dexr_fixed_lag_tape_t* tape = nullptr,
                            const dexr_fixed_lag_accel_t* acc = nullptr) {
  FixedLagArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  a.S = S;
  a.K = K;
  a.flush = io->flush_count_out != nullptr;
  a.wstatus = acc ? fixed_lag_status_words<G, true>(*io, S) : fixed_lag_status_words<G>(*io, S);
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  a.pos_off = round_up(a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4, 16);
  const int smem = a.pos_off + kEvalWarps * 2 * (int)sizeof(long long);
  auto kern = dexr_fixed_lag_kernel<G>;
  auto kern_tape = dexr_fixed_lag_tape_kernel<G>;
  auto kern_acc = dexr_fixed_lag_accel_kernel<G>;
  auto kern_acc_tape = dexr_fixed_lag_accel_tape_kernel<G>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (tape && !acc) CUDA_TRY(cudaFuncSetAttribute(kern_tape, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (acc && !tape) CUDA_TRY(cudaFuncSetAttribute(kern_acc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (acc && tape) CUDA_TRY(cudaFuncSetAttribute(kern_acc_tape, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = (acc && tape) ? eval_ctas_per_sm(kern_acc_tape, smem, &per_sm)
              : acc       ? eval_ctas_per_sm(kern_acc, smem, &per_sm)
                          : eval_ctas_per_sm(kern, smem, &per_sm))
    return e;
  const int grid = (int)std::min<long long>(S, (long long)r->num_sms * per_sm);
  if (acc && tape) kern_acc_tape<<<grid, kEvalWarps * 32, smem, stream>>>(a, *tape, *acc);
  else if (acc) kern_acc<<<grid, kEvalWarps * 32, smem, stream>>>(a, *acc);
  else if (tape) kern_tape<<<grid, kEvalWarps * 32, smem, stream>>>(a, *tape);
  else kern<<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" size_t dexr_fixed_lag_sizeof(void) { return sizeof(dexr_fixed_lag_t); }

extern "C" size_t dexr_fixed_lag_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag) {
  return robot ? fixed_lag_workspace_bytes(robot->host, num_streams, lag) : 0;
}

extern "C" int dexr_fixed_lag_step(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                                   int64_t num_streams, int64_t num_ticks, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step: null argument");
  if (const char* msg = fixed_lag_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || (num_ticks == 0 && !io->flush_count_out)) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_fixed_lag<16>(r, params, io, num_streams, (int)num_ticks, stream)
                                   : launch_fixed_lag<32>(r, params, io, num_streams, (int)num_ticks, stream);
}

extern "C" size_t dexr_fixed_lag_accel_sizeof(void) { return sizeof(dexr_fixed_lag_accel_t); }

extern "C" size_t dexr_fixed_lag_accel_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag) {
  return robot ? fixed_lag_accel_workspace_bytes(robot->host, num_streams, lag) : 0;
}

extern "C" int dexr_fixed_lag_step_accel(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                                         const dexr_fixed_lag_accel_t* acc, int64_t num_streams, int64_t num_ticks,
                                         void* cuda_stream) {
  if (!robot || !params || !io || !acc) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step_accel: null argument");
  if (const char* msg = fixed_lag_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (const char* msg = fixed_lag_accel_error(robot->host, *io, *acc, num_streams)) return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || (num_ticks == 0 && !io->flush_count_out)) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_fixed_lag<16>(r, params, io, num_streams, (int)num_ticks, stream, nullptr, acc)
                                   : launch_fixed_lag<32>(r, params, io, num_streams, (int)num_ticks, stream, nullptr, acc);
}

extern "C" int dexr_fixed_lag_step_accel_tape(const dexr_robot_t* robot, const dexr_params_t* params,
                                              const dexr_fixed_lag_t* io, const dexr_fixed_lag_accel_t* acc,
                                              const dexr_fixed_lag_tape_t* tape, int64_t num_streams, int64_t num_ticks,
                                              void* cuda_stream) {
  if (!robot || !params || !io || !acc || !tape) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step_accel_tape: null argument");
  if (const char* msg = fixed_lag_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (const char* msg = fixed_lag_accel_error(robot->host, *io, *acc, num_streams)) return fail(DEXR_E_INVALID, "%s", msg);
  if (num_ticks > 0)
    if (const char* msg = fixed_lag_tape_error(robot->host, tape)) return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || (num_ticks == 0 && !io->flush_count_out)) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const dexr_fixed_lag_tape_t tp{tape->qpos, robot->host.len_proj > 0 ? tape->projected : nullptr};
  return eval_lanes(r->host) == 16 ? launch_fixed_lag<16>(r, params, io, num_streams, (int)num_ticks, stream, &tp, acc)
                                   : launch_fixed_lag<32>(r, params, io, num_streams, (int)num_ticks, stream, &tp, acc);
}

extern "C" size_t dexr_fixed_lag_tape_sizeof(void) { return sizeof(dexr_fixed_lag_tape_t); }

extern "C" int dexr_fixed_lag_step_tape(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                                        const dexr_fixed_lag_tape_t* tape, int64_t num_streams, int64_t num_ticks,
                                        void* cuda_stream) {
  if (!robot || !params || !io || !tape) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step_tape: null argument");
  if (const char* msg = fixed_lag_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (num_ticks > 0)
    if (const char* msg = fixed_lag_tape_error(robot->host, tape)) return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_params(params)) return e;
  if (num_streams == 0 || (num_ticks == 0 && !io->flush_count_out)) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const dexr_fixed_lag_tape_t tp{tape->qpos, robot->host.len_proj > 0 ? tape->projected : nullptr};
  return eval_lanes(r->host) == 16 ? launch_fixed_lag<16>(r, params, io, num_streams, (int)num_ticks, stream, &tp)
                                   : launch_fixed_lag<32>(r, params, io, num_streams, (int)num_ticks, stream, &tp);
}

// dexr_fixed_lag_step_vjp: launch_fixed_lag's CTA and occupancy rule.  `acc`: dexr_fixed_lag_step_accel_vjp
// (dexr_fixed_lag_accel_vjp_kernel, its own occupancy, the accelerated workspace layout and window view).
template <int G>
static int launch_fixed_lag_vjp(dexr_robot* r, const dexr_params_t* prm, const dexr_fixed_lag_vjp_t* io, long long S, int K,
                                cudaStream_t stream, const dexr_fixed_lag_accel_vjp_t* acc = nullptr) {
  FixedLagVjpArgs a{};
  a.table = r->table_dev;
  a.prm = *prm;
  if (!(io->smooth_weight < 0.f)) a.prm.norm_delta = io->smooth_weight;
  a.io = *io;
  FixedLagPreWs pw{};
  fixed_lag_vjp_layout(r->host, S, io->lag, io->workspace, &a.ws, acc ? &pw : nullptr);
  a.wio = acc ? fixed_lag_accel_vjp_window_io(r->host, a.ws, pw, acc->accel_weight) : fixed_lag_vjp_window_io(r->host, a.ws);
  a.wpk = PackedLayout{a.ws.offsets, 2 * S, S * (io->lag + 1)};
  a.S = S;
  a.K = K;
  a.dm = make_dims(r->host);
  a.scratch_off = round_up((int)sizeof(SharedTable), 16);
  constexpr int GPW = 32 / G;
  a.pos_off = round_up(a.scratch_off + kEvalWarps * GPW * VjpScratch<G>::kFloats * 4, 16);
  const int smem = a.pos_off + kEvalWarps * 2 * (int)sizeof(long long);
  auto kern = dexr_fixed_lag_vjp_kernel<G>;
  auto kern_acc = dexr_fixed_lag_accel_vjp_kernel<G>;
  if (acc) CUDA_TRY(cudaFuncSetAttribute(kern_acc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  else CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 1;
  if (int e = acc ? eval_ctas_per_sm(kern_acc, smem, &per_sm) : eval_ctas_per_sm(kern, smem, &per_sm)) return e;
  const int grid = (int)std::min<long long>(S, (long long)r->num_sms * per_sm);
  if (acc) kern_acc<<<grid, kEvalWarps * 32, smem, stream>>>(a, *acc, pw);
  else kern<<<grid, kEvalWarps * 32, smem, stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  {
    std::lock_guard<std::mutex> lk(r->info_mu);
    r->last = dexr_launch_info_t{grid, kEvalWarps * 32, smem, 0, G, kEvalWarps, r->last.kernels_launched + 1};
  }
  return 0;
}

extern "C" size_t dexr_fixed_lag_vjp_sizeof(void) { return sizeof(dexr_fixed_lag_vjp_t); }

extern "C" size_t dexr_fixed_lag_vjp_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag) {
  return robot ? fixed_lag_vjp_workspace_bytes(robot->host, num_streams, lag) : 0;
}

extern "C" int dexr_fixed_lag_step_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_vjp_t* io,
                                       int64_t num_streams, int64_t num_ticks, void* cuda_stream) {
  if (!robot || !params || !io) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step_vjp: null argument");
  if (const char* msg = fixed_lag_vjp_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_fixed_lag_vjp<16>(r, params, io, num_streams, (int)num_ticks, stream)
                                   : launch_fixed_lag_vjp<32>(r, params, io, num_streams, (int)num_ticks, stream);
}

extern "C" size_t dexr_fixed_lag_accel_vjp_sizeof(void) { return sizeof(dexr_fixed_lag_accel_vjp_t); }

extern "C" size_t dexr_fixed_lag_accel_vjp_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag) {
  return robot ? fixed_lag_accel_vjp_workspace_bytes(robot->host, num_streams, lag) : 0;
}

extern "C" int dexr_fixed_lag_step_accel_vjp(const dexr_robot_t* robot, const dexr_params_t* params,
                                             const dexr_fixed_lag_vjp_t* io, const dexr_fixed_lag_accel_vjp_t* acc,
                                             int64_t num_streams, int64_t num_ticks, void* cuda_stream) {
  if (!robot || !params || !io || !acc) return fail(DEXR_E_INVALID, "dexr_fixed_lag_step_accel_vjp: null argument");
  if (const char* msg = fixed_lag_vjp_io_error(robot->host, *io, *params, num_streams, num_ticks))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (const char* msg = fixed_lag_accel_vjp_error(robot->host, *io, *acc, num_streams))
    return fail(DEXR_E_INVALID, "%s", msg);
  if (int e = check_loss_params(params)) return e;
  if (num_streams == 0) return 0;
  DEVICE_SCOPE(robot->device);
  dexr_robot* r = const_cast<dexr_robot*>(robot);
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  return eval_lanes(r->host) == 16 ? launch_fixed_lag_vjp<16>(r, params, io, num_streams, (int)num_ticks, stream, acc)
                                   : launch_fixed_lag_vjp<32>(r, params, io, num_streams, (int)num_ticks, stream, acc);
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
