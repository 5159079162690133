"""Geman-McClure robustifier of the data rows (oracle; test infrastructure only).

Reference: scan2mesh/robustifiers.py:33-100, ``GMOf`` = SignedSqrt(GMOfInternal(x, sigma)), in closed form; pinned against the
unmodified reference by tests/golden/ref_gmof.npz.  Both stages apply it per coordinate of a visible marker's residual e:
the row becomes wt psi(e) and its Jacobian row the least-squares one times psi'(e).
"""
from __future__ import annotations

import numpy as np


def gm_psi(x, sigma):
    """GMOf(x, sigma) = SignedSqrt(GMOfInternal(x, sigma)) = sigma x / sqrt(sigma^2 + x^2)."""
    x = np.asarray(x, dtype=np.float64)
    return sigma * x / np.sqrt(sigma * sigma + x * x)


def gm_dpsi(x, sigma):
    """d GMOf / dx = (sigma^2 / (sigma^2 + x^2))^(3/2); 0 at x = 0, where the reference's SignedSqrt masks its derivative."""
    x = np.asarray(x, dtype=np.float64)
    t = sigma * sigma / (sigma * sigma + x * x)
    return np.where(x != 0, t * np.sqrt(t), 0.0)
