// emu_fixed_lag.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) running fixed-lag smoothing of the product's dexr_kernels.cuh:
// fixed_lag_tick and fixed_lag_flush on Solver<G, 0> the way dexr_fixed_lag_kernel runs it (a stream's ticks in order on one warp; a 16-lane
// warp's second group idles).
#include "emu_driver.cpp"

namespace {
template <int G>
int run_fixed_lag(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_fixed_lag_t& io, long long S, int K,
                  char* err, int errlen) {
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
        fixed_lag_tick(sv, io, dm, prm, fixed_lag_status_words<G>(io, S), K, pos, lane < G);
      }
      if (io.flush_count_out) fixed_lag_flush(sv, io, dm, prm, s, lane < G);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", s, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// The library's dexr_fixed_lag_workspace_bytes on a host table.
extern "C" size_t emu_fixed_lag_workspace_bytes(const dexr_table_t* tb, long long S, int lag) {
  return fixed_lag_workspace_bytes(*tb, S, lag);
}

// Emulated dexr_fixed_lag_step, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_fixed_lag_step(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_fixed_lag_t* io, long long S,
                                  long long K, char* err, int errlen) {
  if (const char* msg = fixed_lag_io_error(*tb, *io, *prm, S, K)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || (K == 0 && !io->flush_count_out)) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  return eval_lanes(*tb) == 16 ? run_fixed_lag<16>(tb, p, *io, S, (int)K, err, errlen)
                               : run_fixed_lag<32>(tb, p, *io, S, (int)K, err, errlen);
}
