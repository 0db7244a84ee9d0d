"""Coefficients of gelu_erf_fast (pipeedge_b200/csrc/gemm_wgmma.cu): degree-7 fit of log2(erfc(a/sqrt2)/2) on [0, 6]
at Chebyshev nodes, expanded to the power basis, and its error against the exact erf GELU in emulated fp32."""
import numpy as np
from numpy.polynomial import Polynomial, chebyshev as C, polynomial as P
from scipy.special import erf, erfc

A = 6.0
a = np.cos(np.pi * (np.arange(8000) + 0.5) / 8000) * A / 2 + A / 2
f = np.log2(0.5 * erfc(a / np.sqrt(2)))
ch = C.Chebyshev.fit(a, f, 7, domain=[0, A])
t = Polynomial([-1, 2 / A])
T = [Polynomial([1.0]), t]
for k in range(2, 8):
    T.append(2 * t * T[-1] - T[-2])
c = sum((ck * T[k] for k, ck in enumerate(ch.coef)), Polynomial([0.0])).coef
print("max |fit - log2 E| =", np.abs(P.polyval(a, c) - f).max())
print("coefficients c0..c7:", ", ".join(f"{v:.9e}" for v in c))
c32 = c.astype(np.float32)
x = np.linspace(-8, 8, 2000001).astype(np.float32)
ax = np.minimum(np.abs(x), np.float32(A))
p = np.full_like(x, c32[7])
for k in range(6, -1, -1):
    p = (p * ax + c32[k]).astype(np.float32)
e = np.exp2(p.astype(np.float64)).astype(np.float32)
r = (np.maximum(x, 0) - np.abs((x * e).astype(np.float32))).astype(np.float32)
ref = 0.5 * x.astype(np.float64) * (1 + erf(x.astype(np.float64) / np.sqrt(2)))
err = np.abs(r - ref)
print("fp32 emulation: max abs err", err.max(), "max rel err (|x| < 5)", (err / np.maximum(np.abs(ref), 1e-6))[np.abs(x) < 5].max())
