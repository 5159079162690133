"""Development tool (GPU): one small case through the CUDA library (f64 and f32, optional env switches) against the
test-only host build of the same source, frame by frame.  Usage: python tools/gpu_debug_case.py C4"""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import conftest  # noqa: E402
from moshpp_b200 import build, chmosh, lib, synth  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else 'C4'
case = synth.make_case(tempfile.mkdtemp(), name, **conftest.SMALL[name])
pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
case['pack'] = pk
obs, vis = conftest.dense_obs(case)
print(name, 'markers', pk.n_markers, 'n1', len(pk.free_step1), 'n2', len(pk.free_step2), 'joints', pk.n_joints, 'kw', pk.kw)

handle = C.CDLL(build.build_emu())
h = lib.DescHolder(pk)
F = obs.shape[0]
emu = lib.ResultArrays(F, lib.pack_dims(pk))
o64 = np.ascontiguousarray(obs, dtype=np.float64)
v8 = np.ascontiguousarray(vis, dtype=np.uint8)
handle.mosh2_emu_solve(C.byref(h.desc), C.byref(opts), F, o64.ctypes.data_as(lib._f64p), v8.ctypes.data_as(lib._u8p), 0, 0,
                       lib.MOSH2_F64, C.byref(emu.c))
print('emu f64 builds', emu.counters[:, 2].tolist())
for envs in ({}, {'MOSH2_DEV_TILE': '10'}, {'MOSH2_DEV_BIG': '1'}):
    for k in ('MOSH2_DEV_TILE', 'MOSH2_DEV_BIG'):
        os.environ.pop(k, None)
    os.environ.update(envs)
    for prec in ('f64', 'f32'):
        r = conftest.gpu_solve(case, precision=prec)
        dp = np.abs(r.pose - emu.pose).max(axis=1)
        print(envs, prec, 'builds', r.counters[:, 2].tolist(), 'max dpose per frame', np.array2string(dp, precision=2))
