"""mosh2_job_upload_markers_range through the host build of the device source (tests/emu/mosh2_emu_adapter.cpp: the
library's argument checks and mosh2::gather_marker_sample, the function the gather kernel runs per sample): several captures
that differ in column order, unit, rotation and frame range, written into their ranges of one batch frame axis, against the
host adapter (MocapSession.frames_for_labels).  The GPU twin is test_gpu_subject_batch.py."""
import ctypes as C

import numpy as np
import pytest

from moshpp_b200 import build, lib
from moshpp_b200.mocap_interface import MocapSession, load_markers, rotation_xyz

E_INVALID = -1          # MOSH2_E_INVALID


@pytest.fixture(scope='module')
def upload_range():
    f = C.CDLL(build.build_emu()).mosh2_emu_upload_markers_range
    f.argtypes = [C.c_int32, C.c_int32, C.c_int32, lib._f64p, lib._u8p, C.c_int32, C.c_int32, lib._f64p, C.c_int32, C.c_int32,
                  lib._i32p, C.c_int32, C.c_int32, C.c_double, lib._f64p]
    return f


def _call(f, precision, obs, vis, frame0, n, raw, cols, start, step, unit, rot):
    raw = np.ascontiguousarray(raw, dtype=np.float64)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    r = None if rot is None else np.ascontiguousarray(rot, dtype=np.float64)
    return f(precision, obs.shape[1], obs.shape[0], lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p), frame0, n, lib._ptr(raw, lib._f64p),
             raw.shape[0], raw.shape[1], lib._ptr(cols, lib._i32p), start, step, unit, lib._ptr(r, lib._f64p) if r is not None else None)


@pytest.mark.parametrize('precision', [lib.MOSH2_F64, lib.MOSH2_F32])
def test_ranges_equal_host_adapter(cases, tmp_path, upload_range, precision):
    case = cases('C1')           # (c3d, millimetres, NaN gaps, an extra label)
    labels = case['latent_labels']
    raw0, raw_labels, _ = load_markers(case['mocap_fname'])
    specs = []
    for k, (unit, rot, start, step) in enumerate((('mm', None, 0, 1), ('m', None, 2, 2), ('mm', [10.0, -20.0, 30.0], 1, 3))):
        perm = np.random.default_rng(k).permutation(raw0.shape[1])
        mk = raw0[:, perm] / (1000.0 if unit == 'm' else 1.0)
        mk[k::5, perm == 0] = 0.0                               # exact zeros are missing samples too
        fn = str(tmp_path / f'cap{k}.npz')
        np.savez(fn, markers=mk, labels=np.array(raw_labels)[perm], frame_rate=120.0)
        m = MocapSession(fn, unit, mocap_rotate=rot)
        sel = range(start, len(m), step)
        obs, vis = m.frames_for_labels(labels, sel)
        specs.append(dict(m=m, sel=sel, obs=obs, vis=vis, cols=m.raw_columns_for_labels(labels), rot=rot))
    counts = [len(s['sel']) for s in specs]
    off = np.concatenate([[0], np.cumsum(counts)])
    obs = np.full((off[-1], len(labels), 3), np.nan)
    vis = np.full((off[-1], len(labels)), 7, dtype=np.uint8)
    for k, s in enumerate(specs):
        rot = None if s['rot'] is None else rotation_xyz(s['rot'])
        assert _call(upload_range, precision, obs, vis, int(off[k]), counts[k], s['m'].raw, s['cols'], s['sel'].start, s['sel'].step,
                     s['m'].unit_per_metre, rot) == 0
    want_obs = np.concatenate([s['obs'] for s in specs])
    want_vis = np.concatenate([s['vis'] for s in specs])
    assert np.array_equal(vis.astype(bool), want_vis) and set(np.unique(vis)) == {0, 1} and (~want_vis).any()
    if precision == lib.MOSH2_F32:
        want_obs = want_obs.astype(np.float32).astype(np.float64)
    plain = slice(0, int(off[2]))
    assert np.array_equal(obs[plain], want_obs[plain])
    assert np.abs(obs[off[2]:] - want_obs[off[2]:]).max() < (1e-7 if precision == lib.MOSH2_F32 else 1e-12)


def test_range_checks(cases, upload_range):
    raw = np.zeros((10, 4, 3))
    obs, vis = np.zeros((6, 2, 3)), np.zeros((6, 2), dtype=np.uint8)
    cols = [0, 3]
    assert _call(upload_range, 1, obs, vis, 0, 6, raw, cols, 4, 1, 1.0, None) == 0
    assert _call(upload_range, 1, obs, vis, 1, 6, raw, cols, 0, 1, 1.0, None) == E_INVALID    # past the job's frames
    assert _call(upload_range, 1, obs, vis, 0, 6, raw, cols, 5, 1, 1.0, None) == E_INVALID    # past the file's frames
    assert _call(upload_range, 1, obs, vis, 0, 3, raw, cols, 0, 5, 1.0, None) == E_INVALID    # stride past the end
    assert _call(upload_range, 1, obs, vis, 0, 3, raw, [0, 4], 0, 1, 1.0, None) == E_INVALID  # column outside the file
    assert _call(upload_range, 1, obs, vis, 0, 3, raw, cols, 0, 1, 0.0, None) == E_INVALID    # unit
