"""Development tool (CPU): how well-conditioned is the REFERENCE's own result?  Runs the float64 oracle on a window of the
north-star sequence twice -- once as is, once with the observations perturbed by N(0, eps) (eps << the 1 mm marker noise) --
and prints the pose difference per frame."""
import sys, tempfile, time
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np
from make_long_golden import LONG
from moshpp_b200 import synth
from moshpp_b200.mocap_interface import MocapSession
from oracle import stageii
name, kw = LONG['NS']
case = synth.make_case(tempfile.mkdtemp(), name, **kw)
g = np.load(os.path.join(ROOT, 'tests', 'golden', 'long_NS.npz'))
lo, hi = 1300, 1440
def run(eps, seed):
    mocap = MocapSession(case['mocap_fname'], 'mm')
    mocap.markers = mocap.markers[lo:hi].copy()
    if eps:
        rng = np.random.default_rng(seed)
        ok = MocapSession.marker_availability_mask(mocap.markers)
        mocap.markers[ok] += rng.normal(0, eps, mocap.markers[ok].shape)
    out = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'], mocap=mocap)
    return out['_pose_reduced']
A = run(0, 0)
print('cold-started window vs sequential fixture (frames 1400..1439):', np.abs(A[100:] - g['pose'][1400:1440])[:, :66].max(1).round(5).tolist())
for eps in (1e-9, 1e-7, 1e-6):
    B = run(eps, 1)
    d = np.abs(A - B)[:, :66].max(1)
    print(f'eps {eps:g} m: max |dpose| over window {d.max():.2e} at frame {lo + d.argmax()}; frames>1e-3: {(d>1e-3).sum()}; per-frame 1400..1420:', d[100:120].round(5).tolist())
