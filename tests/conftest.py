import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a real H100 (run with -m gpu)')


# small variants of the BASELINE configs: same topology / variable layout, fewer vertices and frames,
# so the float64 oracle finishes in seconds
SMALL = {
    'C1': dict(frames=12, n_verts=1200),
    'C2': dict(frames=16, n_verts=1500),
    'C3': dict(frames=10, n_verts=2000),
    'C4': dict(frames=12, n_verts=None),
    'CF': dict(frames=8, n_verts=2000),       # SMPL-X with face markers: jaw + expressions (SURVEY.md 8(f-4))
    'CH': dict(frames=10, n_verts=1500),      # animal_horse: single-Gaussian pose prior + joint-angle term (SURVEY.md 8(f-4))
}


@pytest.fixture(scope='session')
def case_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp('mosh_cases'))


@pytest.fixture(scope='session')
def cases(case_dir):
    from moshpp_b200 import synth
    cache = {}

    def get(name, **kw):
        key = (name, tuple(sorted(kw.items())))
        if key not in cache:
            args = dict(SMALL.get(name, {}))
            args.update(kw)
            cache[key] = synth.make_case(case_dir, name, **args)
        return cache[key]
    return get


def dense_obs(case):
    from moshpp_b200.mocap_interface import MocapSession
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    return mocap.frames_for_labels(case['latent_labels'], range(len(mocap)))


@pytest.fixture(scope='session')
def emu():
    """TEST-ONLY single-thread host build of the device source (never part of the product)."""
    from moshpp_b200 import build, lib
    handle = C.CDLL(build.build_emu())

    def solve(case, chunk_len=0, warmup=0, precision=None, obs_vis=None, warmup_full=-1, first_extra=0):
        precision = lib.MOSH2_F64 if precision is None else precision
        pk, cfg = case['pack'], case['cfg']
        obs, vis = obs_vis if obs_vis is not None else dense_obs(case)
        h = lib.DescHolder(pk)
        opt = lib.make_options(cfg.opt_settings.weights, optimize_fingers=cfg.moshpp.optimize_fingers and pk.finger_hi > pk.finger_lo,
                               optimize_dynamics=cfg.moshpp.optimize_dynamics,
                               optimize_face=bool(cfg.moshpp.optimize_face) and pk.n_expr > 0)
        F = obs.shape[0]
        res = lib.ResultArrays(F, lib.pack_dims(pk))
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        vis8 = np.ascontiguousarray(vis, dtype=np.uint8)
        sched = lib.make_schedule(chunk_len, warmup, warmup_full, first_extra)
        rc = handle.mosh2_emu_solve(C.byref(h.desc), C.byref(opt), F, obs.ctypes.data_as(lib._f64p),
                                    vis8.ctypes.data_as(lib._u8p), C.byref(sched), precision, C.byref(res.c))
        assert rc == 0
        return res
    return solve


def run_oracle(case, **kw):
    from oracle import stageii
    return stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'],
                                case['betas'], case['marker_meta'], **kw)


def gpu_solve(case, chunk_len=0, warmup=0, precision='f32', obs_vis=None, warmup_full=-1, first_extra=0):
    from moshpp_b200 import chmosh, lib
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'],
                                             case['betas'], case['marker_meta'])
    obs, vis = obs_vis if obs_vis is not None else dense_obs(case)
    model = lib.Model(pk, device=0)
    try:
        return model.solve(obs, vis, opts, chunk_len=chunk_len, chunk_warmup=warmup, warmup_full=warmup_full,
                           precision={'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision], first_extra=first_extra)
    finally:
        model.close()


class EmuStageIBackend:
    """TEST-ONLY back end of moshpp_b200.stagei: the per-frame linearisation through the single-thread host build of the
    device source (mosh2_emu_linearize), the point-to-mesh distances through the oracle (the CUDA kernel has no host build)."""

    def __init__(self):
        from moshpp_b200 import build, lib
        self.lib = lib
        self.handle = C.CDLL(build.build_emu())

    def linearize(self, pk, options, obs, vis, x, step, build):
        lib = self.lib
        F, M = obs.shape[0], pk.n_markers
        n = len(pk.free_step2) if step == 2 else len(pk.free_step1)
        h = lib.DescHolder(pk)
        o = np.ascontiguousarray(obs, dtype=np.float64)
        v8 = np.ascontiguousarray(vis, dtype=np.uint8)
        x = np.ascontiguousarray(x, dtype=np.float64)
        out = dict(errs=np.zeros((F, len(lib.ERR_NAMES))), markers_sim=np.zeros((F, M, 3)), r=np.zeros((F, 3 * M)), vp=np.zeros((F, 3 * M, 3)))
        if build:
            out.update(A=np.zeros((F, n, n)), g=np.zeros((F, n)), J=np.zeros((F, 3 * M, n)))
        c = lib.LinOut(*[lib._ptr(out[k], lib._f64p) if k in out else None for k in ('errs', 'markers_sim', 'r', 'vp', 'A', 'g', 'J')])
        rc = self.handle.mosh2_emu_linearize(C.byref(h.desc), C.byref(options), F, lib._ptr(o, lib._f64p), lib._ptr(v8, lib._u8p),
                                             int(step), int(bool(build)), lib._ptr(x, lib._f64p), C.byref(c))
        assert rc == 0
        return out

    def squared_distance(self, samples, verts, faces):
        from oracle import mesh_distance as omd
        r, ds, dt, tri, part = omd.somedistance(samples, verts, faces, kind=omd.KIND_SQUARED)
        return r, tri, part, ds, dt


def stagei_case(cases, name='C2', n_pick=4, **kw):
    """A Stage-I problem from a synthetic Stage-II case: ``n_pick`` frames of its mocap as label dictionaries."""
    import copy
    from moshpp_b200.mocap_interface import MocapSession
    case = cases(name, **kw)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_betas = True
    mocap = MocapSession(case['mocap_fname'], cfg.mocap.unit)
    frames = mocap.markers_asdict()
    pick = np.linspace(0, len(frames) - 1, n_pick).astype(int)
    return case, cfg, [frames[i] for i in pick]
