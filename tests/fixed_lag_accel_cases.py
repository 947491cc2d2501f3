"""The float64 model of one window solve of acceleration-penalised fixed-lag smoothing (`dexr_fixed_lag_step_accel`),
shared by the host emulation (tests/test_fixed_lag_accel_emulation.py), the GPU suite (tests/test_gpu_fixed_lag_accel.py)
and tools/bench_fixed_lag_accel.py.

`smooth_accel_cases.Model` with the optional pre-anchor p (the frame committed before the anchor a, both clipped): one more
difference row (x_0 - 2 a + p, weight c), so F gains c |x_0 - 2 a + p|^2.  The row's x_0 coefficient puts 2c on x_0's
diagonal block and its share in x_0's gradient; a and p are constants, so nothing else changes.  `polish`, `value`, `grad`
and `hessian` are the base class's, on the extended rows.
"""
import numpy as np

import smooth_accel_cases as SAC
import smooth_cases as SMC

PARITY = SMC.PARITY


class Model(SAC.Model):
    """One window: smooth_accel_cases.Model plus the pre-anchor `pre` (clipped; None: a fresh stream, no such triple)."""

    def __init__(self, o, keypoints, fixed, flags, anchor, w, c, pre=None):
        super().__init__(o, keypoints, fixed, flags, anchor, w, c)
        T = self.T
        self.pre = None if pre is None else np.asarray(pre, np.float64)
        D = np.concatenate([self.D, np.zeros((len(self.D), 1))], 1)  # column T + 1: the pre-anchor
        if self.pre is not None and self.anchor is not None and T > 0:
            r = np.zeros(T + 2)
            r[0], r[T], r[T + 1] = 1.0, -2.0, 1.0
            D = np.vstack([D, r])
            self.Wr = np.append(self.Wr, self.c)
        self.D = D

    def _residuals(self, X):
        a = self.anchor if self.anchor is not None else np.zeros(self.n)
        p = self.pre if self.pre is not None else np.zeros(self.n)
        Y = np.concatenate([np.asarray(X, np.float64).reshape(self.T, self.n), a[None], p[None]])
        return self.D @ Y


def clipped(o, q):
    """clip(q) to clip_lo / clip_hi, as the kernel clips the anchor and the pre-anchor (float64)."""
    return SMC.clipped_anchor(o, q)
