// emu_jacobian.cpp -- TEST INFRASTRUCTURE.  The host emulation of emu_driver.cpp (same fiber warp, shared memory and
// NaN-poisoned scratch, which it includes whole) plus the per-frame Jacobians of the solve: runs the Jacobian driver of the
// product's dexr_kernels.cuh (jacobian_frame on Solver<G, 0>) the way dexr_jacobian_kernel does, one frame per group of G
// lanes.
#include "emu_driver.cpp"

// ---- per-frame Jacobians: jacobian_frame on Solver<G, 0>, the way dexr_jacobian_kernel runs it
namespace {
template <int G>
int run_jacobian(const dexr_table_t* tb, const dexr_params_t& prm, const dexr_jacobian_t& io, long long B, char* err,
                 int errlen) {
  constexpr int GPW = 32 / G;
  const Dims dm = make_dims(*tb);
  const int scratch_off = load_table<0>(tb);
  const int in_row = io.keypoints ? 3 * DEXR_NUM_KEYPOINTS : 3 * dm.n_res;
  for (long long base = 0; base < B; base += GPW) {
    auto lane_body = [&](int lane) {
      Solver<G, 0> sv;
      sv.init(tb, dm, (uint32_t)(scratch_off + lane / G * VjpScratch<G>::kFloats * 4), prm, lane);
      const long long idx = base + lane / G;
      const bool active = idx < B;
      const long long f = active ? idx : base;
      FrameInputs in;
      in.kp = io.keypoints ? io.keypoints + f * in_row : nullptr;
      in.ref = io.keypoints ? nullptr : io.ref_value + f * in_row;
      in.fixed = dm.n_fixed > 0 ? io.fixed_qpos + f * dm.n_fixed : nullptr;
      in.last = nullptr;
      in.projected = nullptr;
      jacobian_frame(sv, in, io, dm, f, active);
    };
    if (int rc = run_poisoned(scratch_off, GPW * VjpScratch<G>::kFloats, lane_body, "frame", base, err, errlen)) return rc;
  }
  return 0;
}
}  // namespace

// Emulated dexr_solve_jacobian, with the library's checks of the arguments that need the table (DEXR_E_INVALID = -1).
extern "C" int emu_solve_jacobian(const dexr_table_t* tb, const dexr_params_t* prm, const dexr_jacobian_t* io, long long B,
                                  char* err, int errlen) {
  if (const char* msg = jacobian_io_error(*tb, *io, *prm)) {
    snprintf(err, errlen, "%s", msg);
    return DEXR_E_INVALID;
  }
  if (B <= 0) return 0;
  return eval_lanes(*tb) == 16 ? run_jacobian<16>(tb, *prm, *io, B, err, errlen)
                               : run_jacobian<32>(tb, *prm, *io, B, err, errlen);
}
