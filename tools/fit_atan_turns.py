"""Fit of the odd minimax polynomial behind lean_atan2_turns (csrc/lean_filter.cuh): atan(t) / 2pi = t P(t^2) on [0, 1], and the
measured fp32 Horner error of each degree (the kernel uses degree 6 in s = t^2).  The errors printed here are sampled; the
bound the classifier charges rests on the exhaustive sweep of tests/cpp/atan_certificate.cu."""
import numpy as np
from numpy.polynomial import chebyshev as C
# fit atan(t)/(2*pi) = t * P(s), s = t^2 on [0,1], minimising max abs error (weighted least squares on Chebyshev nodes, then a few Remez-like reweightings)
def fit(deg):
    N = 4000
    k = np.arange(N)
    t = 0.5 * (1 - np.cos(np.pi * (k + 0.5) / N))  # Chebyshev nodes in [0,1]
    t = t[t > 1e-6]
    s = t * t
    y = np.arctan(t) / (2 * np.pi) / t
    w = np.ones_like(t)
    for it in range(60):
        A = np.vander(s, deg + 1, increasing=True) * (w * t)[:, None]
        c, *_ = np.linalg.lstsq(A, w * t * y, rcond=None)
        err = t * (np.vander(s, deg + 1, increasing=True) @ c) - np.arctan(t) / (2 * np.pi)
        w = w * (1 + 2 * np.abs(err) / np.abs(err).max())
        w /= w.mean()
    return c, np.abs(err).max()
for deg in (5, 6, 7):
    c, e = fit(deg)
    print(deg, e, e * 2 * np.pi)
    c32 = c.astype(np.float32)
    # fp32 Horner with FMA emulation, on 4M random + structured samples
    rng = np.random.default_rng(0)
    tt = np.concatenate([rng.random(4_000_000), np.linspace(0, 1, 1_000_001)]).astype(np.float32)
    s = (tt.astype(np.float64) * tt.astype(np.float64)).astype(np.float32)
    acc = np.full_like(s, c32[-1])
    for ck in c32[-2::-1]:
        acc = (acc.astype(np.float64) * s.astype(np.float64) + np.float64(ck)).astype(np.float32)
    p = (tt.astype(np.float64) * acc.astype(np.float64)).astype(np.float32)
    ref = np.arctan(tt.astype(np.float64)) / (2 * np.pi)
    d = np.abs(p.astype(np.float64) - ref)
    print("   fp32 max abs err turns %.3e  (rad %.3e)" % (d.max(), d.max() * 2 * np.pi), "coeffs", [float(x) for x in c32])
