// emu_fixed_lag_accel.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) running acceleration-penalised fixed-lag smoothing of the product's
// dexr_kernels.cuh: fixed_lag_tick<G, false, true> and fixed_lag_flush<G, true> on Solver<G, 0> the way
// dexr_fixed_lag_accel_kernel runs them (a stream's ticks in order on one warp; a 16-lane warp's second group idles), and
// smooth_packed_stream<G, true, true> on packed clips with a pre-anchor per stream (the window solve on its own).
#include "emu_driver.cpp"

namespace {
template <int G>
int run_fixed_lag_accel(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_fixed_lag_t& io,
                        const dexr_fixed_lag_accel_t& acc, long long S, int K, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long s = 0; s < S; ++s) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      long long pos[2] = {s, 0};  // (the kernel's loop state, one copy per lane here)
      for (int k = 0; k < K; ++k) {
        pos[1] = k;
        fixed_lag_tick<G, false, true>(sv, io, dm, prm, fixed_lag_status_words<G, true>(io, S), K, pos, lane < G, nullptr,
                                       nullptr, &acc);
      }
      if (io.flush_count_out) fixed_lag_flush<G, true>(sv, io, dm, prm, s, lane < G, &acc);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", s, err, errlen)) return rc;
  }
  return 0;
}

template <int G>
int run_smooth_pre(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_smooth_t& io, const PackedLayout& pk,
                   char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long base = 0; base < pk.S; ++base) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      const PackedStream ps = packed_stream(pk, base);
      smooth_packed_stream<G, true, true>(sv, io, dm, prm, ps, lane < G, static_cast<float*>(io.workspace));
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// The library's dexr_fixed_lag_accel_workspace_bytes on a host table.
extern "C" size_t emu_fixed_lag_accel_workspace_bytes(const dexr_table_t* tb, long long S, int lag) {
  return fixed_lag_accel_workspace_bytes(*tb, S, lag);
}

// Emulated dexr_fixed_lag_step_accel, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_fixed_lag_step_accel(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_fixed_lag_t* io,
                                        const dexr_fixed_lag_accel_t* acc, long long S, long long K, char* err, int errlen) {
  const char* msg = fixed_lag_io_error(*tb, *io, *prm, S, K);
  if (!msg) msg = fixed_lag_accel_error(*tb, *io, *acc, S);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || (K == 0 && !io->flush_count_out)) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  return eval_lanes(*tb) == 16 ? run_fixed_lag_accel<16>(tb, p, *io, *acc, S, (int)K, err, errlen)
                               : run_fixed_lag_accel<32>(tb, p, *io, *acc, S, (int)K, err, errlen);
}

// smooth_packed_stream<G, true, true>: dexr_smooth_sequences_packed_accel (c = pre->accel_weight) on packed clips, each
// stream s with the pre-anchor pre->prev_qpos[s] where pre->has_prev[s] is non-zero (the library's argument checks; no
// cost is written: the pre-anchor state takes io.cost_out's place, as in fixed_lag_tick).
extern "C" int emu_smooth_packed_pre_anchor(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_smooth_t* io,
                                            const dexr_fixed_lag_accel_t* pre, const int64_t* offsets, long long S,
                                            long long N, char* err, int errlen) {
  const char* msg = smooth_io_error(*tb, *io, *prm, offsets, S, N);
  if (!msg) msg = smooth_accel_error(*tb, pre->accel_weight, io->workspace, io->workspace_bytes, N);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  dexr_smooth_t aio = *io;
  aio.smooth_weight = pre->accel_weight;  // (the library's launch: w is in p.norm_delta)
  aio.cost_out = reinterpret_cast<float*>(const_cast<dexr_fixed_lag_accel_t*>(pre));  // (pre_anchor_state)
  const PackedLayout pk{offsets, S, N};
  return eval_lanes(*tb) == 16 ? run_smooth_pre<16>(tb, p, aio, pk, err, errlen)
                               : run_smooth_pre<32>(tb, p, aio, pk, err, errlen);
}
