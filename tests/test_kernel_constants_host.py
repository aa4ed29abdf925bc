"""CPU check of the closed-form approximation the CUDA kernels use for the erf GELU of the FC1 epilogue (common.cuh: gelu_erf /
gelu_erf2; constants restated here, numpy emulates the f32 arithmetic).  It bounds the approximation error itself; the kernels are checked
end to end in the -m gpu tests."""
import numpy as np
from scipy.special import erf

F = np.float32


def test_erf_gelu_of_the_fc1_epilogue():
    x = np.linspace(-9, 9, 600001).astype(F)
    z = (np.abs(x) * F(0.70710678118654752440)).astype(F)
    t = (F(1) / (F(0.3275911) * z + F(1))).astype(F)
    poly = (F(1.061405429) * t + F(-1.453152027)).astype(F)
    for c in (1.421413741, -0.284496736, 0.254829592):
        poly = (poly * t + F(c)).astype(F)
    e = np.exp2(((z * z).astype(F) * F(-1.4426950408889634)).astype(F)).astype(F)
    erf_abs = ((-poly * t).astype(F) * e + F(1)).astype(F)
    hx = (F(0.5) * x).astype(F)
    got = (hx * np.copysign(erf_abs, x) + hx).astype(F)
    ref = 0.5 * x.astype(np.float64) * (1 + erf(x.astype(np.float64) / np.sqrt(2)))
    assert np.abs(got - ref).max() < 1e-6, np.abs(got - ref).max()
