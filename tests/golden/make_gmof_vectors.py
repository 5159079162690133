"""Generates tests/golden/ref_gmof.npz: the Geman-McClure robustifier of the UNMODIFIED reference, `GMOf(x, sigma) =
SignedSqrt(GMOfInternal(x, sigma))` (moshpp.scan2mesh.robustifiers, robustifiers.py:33-100), with its derivative, at several
sigma and x.

The module imports `chumpy`; it runs against the forward-only stand-in tests/golden/ref_shim, which is all it needs: `Ch`
subclassing, `on_changed` and `.r`.  The stand-in has no chain rule, so the derivative is composed here from each class's own
`compute_dr_wrt`: d psi / dx = SignedSqrt'(GMOfInternal(x)) * GMOfInternal'(x).

    python tests/golden/make_gmof_vectors.py <moshpp source directory, the one that holds the moshpp package>
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref_src):
    sys.path.insert(0, os.path.join(HERE, 'ref_shim'))
    sys.path.insert(0, ref_src)
    import chumpy as ch                                             # the stand-in
    assert 'ref_shim' in ch.__file__
    from moshpp.scan2mesh import robustifiers as ref_rob            # the reference, unmodified

    # x per sigma: 0, +-1e-9 m, multiples of sigma around 1 and up to 40 sigma (the reference's derivative of GMOfInternal
    # subtracts two nearly equal terms, its relative error grows as (x / sigma)^2 eps: 40 sigma keeps it near 1e-13)
    sigmas = np.array([0.005, 0.01, 0.03, 0.1])
    k = np.array([1e-3, 0.1, 0.5, 0.9, 1.0, 1.1, 2.0, 5.0, 10.0, 40.0])
    xs, psi, dpsi = [], [], []
    for s in sigmas:
        u = np.concatenate([[0.0, 1e-9], s * k])
        x = np.concatenate([-u[:0:-1], u])                          # symmetric, 0 once
        inner = ref_rob.GMOfInternal(x=ch.Ch(x.copy()), sigma=ch.Ch(np.array([s])))
        outer = ref_rob.SignedSqrt(x=ch.Ch(np.asarray(inner.r)))
        d_inner = inner.compute_dr_wrt(inner.x).diagonal()
        with np.errstate(divide='ignore'):
            d_outer = outer.compute_dr_wrt(outer.x).diagonal()
        xs.append(x)
        psi.append(np.asarray(outer.r))
        dpsi.append(d_outer * d_inner)
    np.savez_compressed(os.path.join(HERE, 'ref_gmof.npz'), x=np.array(xs), sigma=sigmas, psi=np.array(psi), dpsi=np.array(dpsi))
    print('ref_gmof.npz:', len(sigmas), 'sigmas x', len(xs[0]), 'points')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
