// emu_smooth_accel.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) running the acceleration-penalised smoother and its backpropagation of the
// product's dexr_kernels.cuh: smooth_packed_stream<G, true> and smooth_vjp_packed_stream<G, true> on Solver<G, 0> the way
// dexr_smooth_accel_kernel and dexr_smooth_accel_vjp_kernel run them (one stream per warp; a 16-lane warp's second group
// idles).  accel_weight == 0 runs the velocity-only code, as the library's entry points do.
#include "emu_driver.cpp"

namespace {
template <int G, bool ACC>
int run_smooth_accel(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_smooth_t& io,
                     const PackedLayout& pk, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long base = 0; base < pk.S; ++base) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      const PackedStream ps = packed_stream(pk, base);
      smooth_packed_stream<G, ACC>(sv, io, dm, prm, ps, lane < G, static_cast<float*>(io.workspace));
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}

template <int G, bool ACC>
int run_smooth_accel_vjp(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_smooth_vjp_t& io,
                         const PackedLayout& pk, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long base = 0; base < pk.S; ++base) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      smooth_vjp_packed_stream<G, ACC>(sv, io, dm, pk, base, lane < G);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// The library's dexr_smooth_accel_workspace_bytes on a host table.
extern "C" size_t emu_smooth_accel_workspace_bytes(const dexr_table_t* tb, long long N) {
  return smooth_accel_workspace_bytes(*tb, N);
}

// Emulated dexr_smooth_sequences_packed_accel, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_smooth_sequences_packed_accel(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_smooth_t* io,
                                                 float accel, const int64_t* offsets, long long S, long long N, char* err,
                                                 int errlen) {
  const char* msg = smooth_io_error(*tb, *io, *prm, offsets, S, N);
  if (!msg && accel != 0.f) msg = smooth_accel_error(*tb, accel, io->workspace, io->workspace_bytes, N);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  const PackedLayout pk{offsets, S, N};
  if (accel == 0.f)
    return eval_lanes(*tb) == 16 ? run_smooth_accel<16, false>(tb, p, *io, pk, err, errlen)
                                 : run_smooth_accel<32, false>(tb, p, *io, pk, err, errlen);
  dexr_smooth_t aio = *io;
  aio.smooth_weight = accel;  // (the library's launch: w is in p.norm_delta)
  return eval_lanes(*tb) == 16 ? run_smooth_accel<16, true>(tb, p, aio, pk, err, errlen)
                               : run_smooth_accel<32, true>(tb, p, aio, pk, err, errlen);
}

// Emulated dexr_smooth_sequences_packed_accel_vjp, with the library's argument checks.
extern "C" int emu_smooth_sequences_packed_accel_vjp(const dexr_table_t* tb, const dexr_params_t* prm,
                                                     const dexr_smooth_vjp_t* io, float accel, const int64_t* offsets,
                                                     long long S, long long N, char* err, int errlen) {
  const char* msg = smooth_vjp_io_error(*tb, *io, *prm, offsets, S, N);
  if (!msg && accel != 0.f) msg = smooth_accel_error(*tb, accel, io->workspace, io->workspace_bytes, N);
  if (msg) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  const PackedLayout pk{offsets, S, N};
  if (accel == 0.f)
    return eval_lanes(*tb) == 16 ? run_smooth_accel_vjp<16, false>(tb, p, *io, pk, err, errlen)
                                 : run_smooth_accel_vjp<32, false>(tb, p, *io, pk, err, errlen);
  dexr_smooth_vjp_t aio = *io;
  aio.smooth_weight = accel;  // (the library's launch: w is in p.norm_delta)
  return eval_lanes(*tb) == 16 ? run_smooth_accel_vjp<16, true>(tb, p, aio, pk, err, errlen)
                               : run_smooth_accel_vjp<32, true>(tb, p, aio, pk, err, errlen);
}
