// emu_fixed_lag_accel_vjp.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory
// and NaN-poisoned scratch, which it includes whole) running the recording acceleration-penalised fixed-lag forward and the
// backpropagation through it of the product's dexr_kernels.cuh: fixed_lag_tick<G, true, true> / fixed_lag_flush<G, true>
// the way dexr_fixed_lag_accel_tape_kernel runs them, and fixed_lag_vjp_begin / fixed_lag_vjp_rebuild /
// smooth_vjp_packed_stream<G, true, true> / fixed_lag_vjp_scatter with ACC the way dexr_fixed_lag_accel_vjp_kernel runs them
// (a stream's ticks in reverse on one warp; a 16-lane warp's second group idles).
#include "emu_driver.cpp"

namespace {
template <int G>
int run_fixed_lag_accel_tape(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_fixed_lag_t& io,
                             const dexr_fixed_lag_accel_t& acc, const dexr_fixed_lag_tape_t& tape, long long S, int K,
                             char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long s = 0; s < S; ++s) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      long long pos[2] = {s, 0};
      for (int k = 0; k < K; ++k) {
        pos[1] = k;
        fixed_lag_tick<G, true, true>(sv, io, dm, prm, fixed_lag_status_words<G, true>(io, S), K, pos, lane < G, tape.qpos,
                                      tape.projected, &acc);
      }
      if (io.flush_count_out) fixed_lag_flush<G, true>(sv, io, dm, prm, s, lane < G, &acc);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", s, err, errlen)) return rc;
  }
  return 0;
}

template <int G>
int run_fixed_lag_accel_vjp(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_fixed_lag_vjp_t& io,
                            const dexr_fixed_lag_accel_vjp_t& acc, long long S, int K, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  FixedLagVjpWs ws;
  FixedLagPreWs pw;
  fixed_lag_vjp_layout(*tb, S, io.lag, io.workspace, &ws, &pw);
  const dexr_smooth_vjp_t wio = fixed_lag_accel_vjp_window_io(*tb, ws, pw, acc.accel_weight);
  const PackedLayout wpk{ws.offsets, 2 * S, S * (io.lag + 1)};
  for (long long s = 0; s < S; ++s) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      fixed_lag_vjp_begin<G, true>(sv, io, ws, dm, s, K, lane < G, &acc, &pw);
      long long pos[2] = {s, 0};
      for (int k = K - 1; k >= 0; --k) {
        pos[1] = k;
        if (fixed_lag_vjp_rebuild<G, true>(sv, io, ws, dm, K, pos, lane < G, &acc, &pw)) {
          smooth_vjp_packed_stream<G, true, true>(sv, wio, dm, wpk, 2 * pos[0], lane < G);
          fixed_lag_vjp_scatter<G, true>(sv, io, ws, dm, K, pos, lane < G, &acc, &pw);
        }
      }
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", s, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// The library's dexr_fixed_lag_accel_vjp_workspace_bytes on a host table.
extern "C" size_t emu_fixed_lag_accel_vjp_workspace_bytes(const dexr_table_t* tb, long long S, int lag) {
  return fixed_lag_accel_vjp_workspace_bytes(*tb, S, lag);
}

// Emulated dexr_fixed_lag_step_accel_tape, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_fixed_lag_step_accel_tape(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_fixed_lag_t* io,
                                             const dexr_fixed_lag_accel_t* acc, const dexr_fixed_lag_tape_t* tape, long long S,
                                             long long K, char* err, int errlen) {
  const char* msg = fixed_lag_io_error(*tb, *io, *prm, S, K);
  if (!msg) msg = fixed_lag_accel_error(*tb, *io, *acc, S);
  if (!msg && K > 0) msg = fixed_lag_tape_error(*tb, tape);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || (K == 0 && !io->flush_count_out)) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  const dexr_fixed_lag_tape_t tp{tape->qpos, tb->len_proj > 0 ? tape->projected : nullptr};
  return eval_lanes(*tb) == 16 ? run_fixed_lag_accel_tape<16>(tb, p, *io, *acc, tp, S, (int)K, err, errlen)
                               : run_fixed_lag_accel_tape<32>(tb, p, *io, *acc, tp, S, (int)K, err, errlen);
}

// Emulated dexr_fixed_lag_step_accel_vjp, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_fixed_lag_step_accel_vjp(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_fixed_lag_vjp_t* io,
                                            const dexr_fixed_lag_accel_vjp_t* acc, long long S, long long K, char* err,
                                            int errlen) {
  const char* msg = fixed_lag_vjp_io_error(*tb, *io, *prm, S, K);
  if (!msg) msg = fixed_lag_accel_vjp_error(*tb, *io, *acc, S);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  return eval_lanes(*tb) == 16 ? run_fixed_lag_accel_vjp<16>(tb, p, *io, *acc, S, (int)K, err, errlen)
                               : run_fixed_lag_accel_vjp<32>(tb, p, *io, *acc, S, (int)K, err, errlen);
}

// sizeof(dexr_fixed_lag_accel_vjp_t) and sizeof(dexr_fixed_lag_vjp_t) as the library sees them.
extern "C" size_t emu_fixed_lag_accel_vjp_sizeof(void) { return sizeof(dexr_fixed_lag_accel_vjp_t); }
extern "C" size_t emu_fixed_lag_vjp_sizeof(void) { return sizeof(dexr_fixed_lag_vjp_t); }
