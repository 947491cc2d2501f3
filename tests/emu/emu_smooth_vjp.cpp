// emu_smooth_vjp.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) running the backpropagation through the offline smoother of the product's
// dexr_kernels.cuh: smooth_vjp_packed_stream on Solver<G, 0> the way dexr_smooth_vjp_kernel runs it (one stream per warp;
// a 16-lane warp's second group idles).
#include "emu_driver.cpp"

namespace {
template <int G>
int run_smooth_vjp(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_smooth_vjp_t& io, const PackedLayout& pk,
                   char* err, int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  for (long long base = 0; base < pk.S; ++base) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      smooth_vjp_packed_stream(sv, io, dm, pk, base, lane < G);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// Emulated dexr_smooth_sequences_packed_vjp, with the library's argument checks (DEXR_E_INVALID = -1).
extern "C" int emu_smooth_sequences_packed_vjp(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_smooth_vjp_t* io,
                                               const int64_t* offsets, long long S, long long N, char* err, int errlen) {
  if (const char* msg = smooth_vjp_io_error(*tb, *io, *prm, offsets, S, N)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  dexr_params_t p = *prm;
  if (!(io->smooth_weight < 0.f)) p.norm_delta = io->smooth_weight;
  const PackedLayout pk{offsets, S, N};
  return eval_lanes(*tb) == 16 ? run_smooth_vjp<16>(tb, p, *io, pk, err, errlen) : run_smooth_vjp<32>(tb, p, *io, pk, err, errlen);
}
