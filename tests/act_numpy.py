"""TEST INFRASTRUCTURE ONLY (CPU, numpy float64): the activation derivatives of the extended kernel instances (PJ_ACT_SIGMOID,
PJ_ACT_SILU, PJ_ACT_ELU) for the numpy mirrors of the kernels' algorithm (oracle/jet_numpy.py, tests/jet3_numpy.py).

``install(monkeypatch)`` replaces the mirrors' ``act_derivs`` / ``act_derivs4`` by ``act_derivs4`` below for the duration of a
test: tanh and sine give what the mirrors give, the new codes their exact derivatives in float64.  Never imported by the
product.
"""
import numpy as np

import jet3_numpy
from oracle import jet_numpy

ACT_SIGMOID, ACT_SILU, ACT_ELU = 2, 3, 4
_TANH_SIN = jet3_numpy.act_derivs4


def sigmoid_derivs4(z0):
    """sigmoid(z0) and its first four derivatives, as polynomials in sigmoid(z0)"""
    s = 0.5 * (1.0 + np.tanh(0.5 * z0))   # no overflow of exp(-z0)
    d1 = s * (1.0 - s)
    return s, d1, d1 * (1.0 - 2.0 * s), d1 * (1.0 - 6.0 * s + 6.0 * s * s), d1 * (1.0 - 2.0 * s) * (1.0 - 12.0 * s + 12.0 * s * s)


def act_derivs4(act, z0):
    """value and first four derivatives of activation ``act`` (PJ_ACT_*) at z0"""
    if act in (0, 1):
        return _TANH_SIN(act, z0)
    if act == ACT_SIGMOID:
        return sigmoid_derivs4(z0)
    if act == ACT_SILU:   # (z s)^(k) = k s^(k-1) + z s^(k)
        s = sigmoid_derivs4(z0)
        return (z0 * s[0],) + tuple(k * s[k - 1] + z0 * s[k] for k in range(1, 5))
    if act == ACT_ELU:    # alpha = 1; at z0 = 0: s1 = 1 and higher derivatives 0, as torch's autograd gives them
        pos = z0 >= 0
        e = np.exp(np.minimum(z0, 0.0))
        zero = np.zeros_like(z0)
        return (np.where(pos, z0, np.expm1(np.minimum(z0, 0.0))), np.where(pos, 1.0, e), np.where(pos, zero, e),
                np.where(pos, zero, e), np.where(pos, zero, e))
    raise ValueError(f"unknown activation code {act}")


def act_derivs(act, z0):
    return act_derivs4(act, z0)[:4]


def install(monkeypatch):
    monkeypatch.setattr(jet_numpy, "act_derivs", act_derivs)
    monkeypatch.setattr(jet3_numpy, "act_derivs4", act_derivs4)
