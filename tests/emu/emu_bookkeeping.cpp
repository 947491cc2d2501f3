// emu_bookkeeping.cpp -- TEST INFRASTRUCTURE.  Checks the packed solver bookkeeping of the product's dexr_kernels.cuh
// (Bookkeeping<true>, two 32-bit words, run by the block-diagonal solver) against the unpacked one (Bookkeeping<false>, one
// variable each, run by the dense and arrow solvers): random sequences of the operations Solver::solve applies, with the
// packed-only near-step flag set and cleared in between, must read back the same state after every operation.  The header is
// compiled through emu_driver.cpp (warp shim, shared-memory buffer), which this file includes whole.
#include "emu_driver.cpp"

#include <cstring>
#include <random>

namespace {
int fail(char* err, int errlen, unsigned seed, int step, const char* what, long long packed, long long unpacked) {
  std::snprintf(err, errlen, "seed %u, operation %d: %s differs: packed %lld, unpacked %lld", seed, step, what, packed,
                unpacked);
  return 1;
}
}  // namespace

extern "C" int emu_bookkeeping_check(unsigned seed, int n_ops, char* err, int errlen) {
  using namespace dexr;
  std::mt19937 rng(seed);
  Bookkeeping<true> pk;
  Bookkeeping<false> up;
  bool near_ref = false;
  int rechecks = 0;
  const int flags[3] = {DEXR_STATUS_NOISEFLOOR, DEXR_STATUS_MAXITER, DEXR_STATUS_NONFINITE};
  for (int step = 0; step < n_ops; ++step) {
    const int op = (int)(rng() % 12u);
    const bool b = (rng() & 1u) != 0u;
    switch (op) {
      case 0: pk.inc_iters(); up.inc_iters(); break;
      case 1: pk.inc_rejects(); up.inc_rejects(); break;
      case 2: pk.set_done(b); up.set_done(b); break;
      case 3: pk.set_exact(b); up.set_exact(b); break;
      case 4: pk.set_recheck(b); up.set_recheck(b); break;
      case 5: pk.set_trust_prev(b); up.set_trust_prev(b); break;
      case 6: { const int f = flags[rng() % 3u]; pk.flag(f); up.flag(f); break; }
      case 7: if (b) { pk.clear_stall(); up.clear_stall(); } else { pk.inc_stall(); up.inc_stall(); } break;
      case 8: { const unsigned m = rng() & 0xffffu; pk.set_last_fmask(m); up.set_last_fmask(m); break; }
      case 9:  // solve() counts at most three rechecks per frame (the third ends it)
        if (rechecks < 3) {
          ++rechecks;
          const int a = pk.inc_rechecks(), c = up.inc_rechecks();
          if (a != c) return fail(err, errlen, seed, step, "inc_rechecks()", a, c);
        }
        break;
      default: pk.set_near(b); near_ref = b; break;  // packed only: the unpacked solver keeps the accepted step itself
    }
    if (pk.done() != up.done()) return fail(err, errlen, seed, step, "done()", pk.done(), up.done());
    if (pk.exact() != up.exact()) return fail(err, errlen, seed, step, "exact()", pk.exact(), up.exact());
    if (pk.recheck() != up.recheck()) return fail(err, errlen, seed, step, "recheck()", pk.recheck(), up.recheck());
    if (pk.trust_prev() != up.trust_prev()) return fail(err, errlen, seed, step, "trust_prev()", pk.trust_prev(), up.trust_prev());
    if (pk.iters() != up.iters()) return fail(err, errlen, seed, step, "iters()", pk.iters(), up.iters());
    if (pk.status() != up.status()) return fail(err, errlen, seed, step, "status()", pk.status(), up.status());
    if (pk.last_fmask() != up.last_fmask()) return fail(err, errlen, seed, step, "last_fmask()", pk.last_fmask(), up.last_fmask());
    const int su = up.stall() < 3 ? up.stall() : 3;  // the packed counter saturates at 3: only `stall() >= 2` is read
    if (pk.stall() != su) return fail(err, errlen, seed, step, "stall()", pk.stall(), su);
    if (pk.near() != near_ref) return fail(err, errlen, seed, step, "near()", pk.near(), near_ref);
  }
  return 0;
}

// The sequence of solve() that reaches a recheck with a changed free-variable set: an accepted step below the tolerance with
// a bound active (set_recheck and, the step being below kNearStep as well, set_near), then the next iteration's new mask.
// Returns what inc_rechecks() returns there (1: the first recheck, as in the unpacked solver).
extern "C" int emu_bookkeeping_first_recheck() {
  dexr::Bookkeeping<true> pk;
  pk.set_last_fmask(0x0fffu);
  pk.set_recheck(true);
  pk.set_near(true);
  pk.inc_iters();
  return pk.inc_rechecks();
}
