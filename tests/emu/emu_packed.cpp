// emu_packed.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) running the packed-stream drivers of the product's dexr_kernels.cuh:
// solve_packed_stream<G, BW, REC> the way dexr_packed_sequences_kernel runs it (two 16-lane streams per warp, one 32-lane
// stream, or duo mode: both half-warps on one stream), and vjp_packed_stream the way dexr_packed_seq_vjp_kernel does.
#include "emu_driver.cpp"

namespace {
template <int G, int BW>
int run_packed(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_sequences_t& io, const dexr_sequences_tape_t& tape,
               bool rec, const PackedLayout& pk, bool duo, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  duo = duo && G == 16;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<BW>(tb);
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  for (long long base = 0; base < pk.S; base += duo ? 1 : GPW) {
    auto lane_body = [&](int lane) {
      const int gid = lane / G;
      const uint32_t off = (uint32_t)(scratch_off + gid * Scratch<G>::kStreamFloats * 4);
      Solver<G, BW> sv;
      sv.init(tb, dm, off, prm, lane);
      if (duo) sv.duo = gid;
      const PackedStream ps = packed_stream(pk, duo ? base : base + gid);
      float* kpbuf = reinterpret_cast<float*>(dsmem + off) + Scratch<G>::kFloats;
      const bool owner = !duo || gid == 0;
      if (rec)
        solve_packed_stream<G, BW, true>(sv, io, dm, prm, ps, true, owner, kpbuf, use_filter, tape.qpos, tape.projected);
      else
        solve_packed_stream<G, BW, false>(sv, io, dm, prm, ps, true, owner, kpbuf, use_filter, nullptr, nullptr);
    };
    if (int rc = run_poisoned(scratch_off, GPW * Scratch<G>::kStreamFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}

// `spw` streams per warp: 32 / G, or 1 (the second 16-lane group has no stream).
template <int G>
int run_packed_vjp(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_sequences_vjp_t& io, const PackedLayout& pk,
                   int spw, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  if (spw != 1) spw = GPW;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  for (long long base = 0; base < pk.S; base += spw) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      const bool owner = spw == GPW || lane < G;
      const PackedStream ps = packed_stream(pk, base + (spw == GPW ? lane / G : 0));
      vjp_packed_stream(sv, io, dm, ps, owner, use_filter);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// Emulated dexr_solve_sequences_packed (use_arrow in place of DEXR_ARROW), with the library's argument checks
// (DEXR_E_INVALID = -1).  `tape` NULL: not recorded.
extern "C" int emu_solve_sequences_packed(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow,
                                          const dexr_sequences_t* io, const dexr_sequences_tape_t* tape,
                                          const int64_t* offsets, long long S, long long N, int duo,
                                          char* err, int errlen) {
  if (const char* msg = packed_io_error(*tb, *io, tape, *prm, offsets, S, N)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  const dexr_params_t sp = sequence_params(*prm);
  dexr_sequences_tape_t tp{nullptr, nullptr};
  if (tape) tp = dexr_sequences_tape_t{tape->qpos, tb->loss == DEXR_LOSS_DEXPILOT ? tape->projected : nullptr};
  const PackedLayout pk{offsets, S, N};
  return with_solver(solver_kind(*tb, use_arrow), [&](auto s) {
    return run_packed<decltype(s)::G, decltype(s)::BW>(tb, sp, *io, tp, tape != nullptr, pk, duo != 0, err, errlen);
  });
}

// Emulated dexr_solve_sequences_packed_vjp, with the library's argument checks.
extern "C" int emu_solve_sequences_packed_vjp(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_sequences_vjp_t* io,
                                              const int64_t* offsets, long long S, long long N, int spw,
                                              char* err, int errlen) {
  if (const char* msg = packed_io_error(*tb, *io, *prm, offsets, S, N)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S == 0 || N == 0) return 0;
  const dexr_params_t sp = sequence_params(*prm);
  const PackedLayout pk{offsets, S, N};
  return eval_lanes(*tb) == 16 ? run_packed_vjp<16>(tb, sp, *io, pk, spw, err, errlen)
                               : run_packed_vjp<32>(tb, sp, *io, pk, spw, err, errlen);
}
