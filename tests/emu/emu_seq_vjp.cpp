// emu_seq_vjp.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) plus backpropagation through the sequence solve: runs the recorded stream
// driver (solve_stream<G, BW, true>) the way dexr_sequences_tape_kernel does, and the reverse-time VJP driver of the
// product's dexr_kernels.cuh (vjp_stream on Solver<G, 0>) the way dexr_seq_vjp_kernel does, one stream per group of G lanes.
#include "emu_driver.cpp"

namespace {
// dexr_sequences_tape_kernel with one warp, as run_streams runs dexr_sequences_kernel.
template <int G, int BW>
int run_streams_tape(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_sequences_t& io,
                     const dexr_sequences_tape_t& tape, long long S, int T, bool duo, char* err, int errlen) {
  constexpr int GPW = 32 / G;
  duo = duo && G == 16;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<BW>(tb);
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  for (long long base = 0; base < S; base += duo ? 1 : GPW) {
    auto lane_body = [&](int lane) {
      const int gid = lane / G;
      const uint32_t off = (uint32_t)(scratch_off + gid * Scratch<G>::kStreamFloats * 4);
      Solver<G, BW> sv;
      sv.init(tb, dm, off, prm, lane);
      if (duo) sv.duo = gid;
      const long long s = duo ? base : base + gid;
      float* kpbuf = reinterpret_cast<float*>(dsmem + off) + Scratch<G>::kFloats;
      solve_stream<G, BW, true>(sv, io, dm, prm, S, T, s, s < S, s < S && (!duo || gid == 0), kpbuf, use_filter, tape.qpos,
                                tape.projected);
    };
    if (int rc = run_poisoned(scratch_off, GPW * Scratch<G>::kStreamFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}

// dexr_seq_vjp_kernel with one warp: `spw` streams per warp (32 / G, or 1: the second 16-lane group walks stream S - 1
// inactive).
template <int G>
int run_seq_vjp(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_sequences_vjp_t& io, long long S, int T, int spw,
                char* err, int errlen) {
  constexpr int GPW = 32 / G;
  if (spw != 1) spw = GPW;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  const bool use_filter = prm.lp_alpha >= 0.f && prm.lp_alpha <= 1.f;
  for (long long base = 0; base < S; base += spw) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      const bool owner = spw == GPW || lane < G;
      const long long s = base + (spw == GPW ? lane / G : 0);
      vjp_stream(sv, io, dm, S, T, s, owner && s < S, use_filter);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "stream", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// Emulated dexr_solve_sequences_tape (use_arrow in place of DEXR_ARROW).
extern "C" int emu_solve_sequences_tape(const dexr_table_t* tb, const dexr_params_t* prm, int use_arrow,
                                        const dexr_sequences_t* io, const dexr_sequences_tape_t* tape, long long S,
                                        long long T, int duo, char* err, int errlen) {
  if (S <= 0 || T <= 0) return 0;
  const dexr_params_t sp = sequence_params(*prm);
  const dexr_sequences_tape_t tp{tape->qpos, tb->loss == DEXR_LOSS_DEXPILOT ? tape->projected : nullptr};
  return with_solver(solver_kind(*tb, use_arrow), [&](auto s) {
    return run_streams_tape<decltype(s)::G, decltype(s)::BW>(tb, sp, *io, tp, S, (int)T, duo != 0, err, errlen);
  });
}

// Emulated dexr_solve_sequences_vjp, with the library's checks of the arguments that need the table (DEXR_E_INVALID = -1).
extern "C" int emu_solve_sequences_vjp(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_sequences_vjp_t* io,
                                       long long S, long long T, int spw, char* err, int errlen) {
  if (const char* msg = seq_vjp_io_error(*tb, *io, *prm)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (S <= 0 || T <= 0) return 0;
  const dexr_params_t sp = sequence_params(*prm);
  return eval_lanes(*tb) == 16 ? run_seq_vjp<16>(tb, sp, *io, S, (int)T, spw, err, errlen)
                               : run_seq_vjp<32>(tb, sp, *io, S, (int)T, spw, err, errlen);
}
