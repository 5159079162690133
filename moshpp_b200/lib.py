"""ctypes binding of ``libmosh2.so`` (C-ABI: include/mosh2.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``moshpp_b200/build.py``.  There is no
CPU fallback: if the shared object or a CUDA device is missing, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np

from .pack import StageIIPack

ABI_VERSION = 110          # MOSH2_VERSION of include/mosh2.h that the ctypes structs below encode
MOSH2_F32, MOSH2_F64 = 0, 1
ST_SOLVED, ST_SKIPPED, ST_HAS_VELO, ST_HAS_EXTRAP, ST_GN_FALLBACK, ST_MAXITER, ST_SHORT_WARMUP = 1, 2, 4, 8, 16, 32, 64
ERR_NAMES = ('data', 'poseB', 'velo', 'poseH', 'dmpl', 'extrap_dmpl', 'poseF', 'expr')   # column order of mosh2_result.errs

_i32p = C.POINTER(C.c_int32)
_u8p = C.POINTER(C.c_uint8)
_f64p = C.POINTER(C.c_double)


class ModelDesc(C.Structure):
    _fields_ = [
        ('n_joints', C.c_int32), ('n_markers', C.c_int32), ('body_dof', C.c_int32), ('p_red', C.c_int32),
        ('n_hand_red', C.c_int32), ('n_hand_full', C.c_int32), ('n_dmpl', C.c_int32),
        ('kw', C.c_int32),
        ('parents', _i32p), ('w_joint', _i32p),
        ('hand_comps', _f64p), ('hands_mean', _f64p), ('v0', _f64p), ('sd', _f64p), ('pd', _f64p),
        ('w_val', _f64p), ('j0', _f64p), ('jd', _f64p), ('coefs', _f64p),
        ('prior_k', C.c_int32), ('prior_d', C.c_int32), ('prior_off', C.c_int32), ('prior_ids', _i32p),
        ('prior_means', _f64p), ('prior_Q', _f64p), ('prior_neglogw', _f64p),
        ('n_free1', C.c_int32), ('n_free2', C.c_int32), ('free1', _i32p), ('free2', _i32p),
        ('finger_lo', C.c_int32), ('finger_hi', C.c_int32),
        ('n_expr', C.c_int32), ('face_lo', C.c_int32), ('face_hi', C.c_int32),
        ('n_jangles', C.c_int32), ('jangles_ids', _i32p), ('jangles_signs', _f64p),
    ]


class Options(C.Structure):
    _fields_ = [
        ('wt_data', C.c_double), ('wt_poseB', C.c_double), ('wt_poseH', C.c_double), ('wt_velo', C.c_double),
        ('wt_dmpl', C.c_double), ('wt_annealing', C.c_double), ('wt_extrap_dmpl', C.c_double),
        ('num_train_markers', C.c_double), ('delta_0', C.c_double), ('e3_first', C.c_double), ('e3', C.c_double),
        ('maxiter', C.c_int32), ('optimize_fingers', C.c_int32), ('optimize_dynamics', C.c_int32),
        ('wt_poseF', C.c_double), ('wt_expr', C.c_double), ('optimize_face', C.c_int32),
        ('robust_sigma', C.c_double),
    ]


class Schedule(C.Structure):
    """mosh2_schedule: chunk_len <= 0 = the reference's sequential pass; warmup_full < 0 = every warm-up frame runs
    the full per-frame schedule; first_extra = frames the first chunk of every sequence emits on top of chunk_len (it has
    no warm-up to solve)."""
    _fields_ = [('chunk_len', C.c_int32), ('chunk_warmup', C.c_int32), ('warmup_full', C.c_int32), ('first_extra', C.c_int32)]


def make_schedule(chunk_len: int = 0, chunk_warmup: int = 0, warmup_full: int = -1, first_extra: int = 0) -> Schedule:
    return Schedule(int(chunk_len), int(chunk_warmup), int(warmup_full), int(first_extra))


class Result(C.Structure):
    _fields_ = [
        ('fullpose', _f64p), ('pose', _f64p), ('trans', _f64p), ('dmpls', _f64p), ('markers_sim', _f64p),
        ('errs', _f64p), ('status', _i32p), ('counters', _i32p),
    ]


class MeshDistanceOut(C.Structure):
    _fields_ = [('value', _f64p), ('tri', _i32p), ('part', _i32p), ('d_sample', _f64p), ('d_tri', _f64p)]


class LinOut(C.Structure):
    _fields_ = [('errs', _f64p), ('markers_sim', _f64p), ('r', _f64p), ('vp', _f64p), ('A', _f64p), ('g', _f64p), ('J', _f64p)]


class Mosh2Error(RuntimeError):
    pass


def default_library_path() -> str:
    # MOSH2_LIBRARY: development override (instrumented builds of the same CUDA source)
    return os.environ.get('MOSH2_LIBRARY') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libmosh2.so')


_LIB = None


def load_library(path: Optional[str] = None):
    """Loads libmosh2.so (once) and declares the prototypes of include/mosh2.h."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    p = path or default_library_path()
    if not os.path.exists(p):
        raise Mosh2Error(f'{p} not found: build it with `python -m moshpp_b200.build` (nvcc, sm_90a). '
                         'moshpp_b200 has no CPU solver.')
    lib = C.CDLL(p)
    vp = C.c_void_p
    lib.mosh2_version.restype = C.c_int
    if lib.mosh2_version() != ABI_VERSION:
        raise Mosh2Error(f'{p} implements ABI {lib.mosh2_version()}, this binding encodes {ABI_VERSION}: '
                         'rebuild it with `python -m moshpp_b200.build --force`')
    lib.mosh2_last_error.restype = C.c_char_p
    lib.mosh2_device_count.restype = C.c_int
    lib.mosh2_default_options.argtypes = [C.POINTER(Options)]
    lib.mosh2_default_options.restype = None
    lib.mosh2_release_cached_memory.argtypes = []
    lib.mosh2_mesh_distance.argtypes = [C.c_int32, C.c_int32, C.c_double, C.c_int32, _f64p, C.c_int32, _f64p, C.c_int32, _i32p, _i32p,
                                        _i32p, C.POINTER(MeshDistanceOut), C.POINTER(C.c_float)]
    lib.mosh2_release_cached_memory.restype = None
    lib.mosh2_model_create.argtypes = [C.POINTER(ModelDesc), C.c_int, C.POINTER(vp)]
    lib.mosh2_model_destroy.argtypes = [vp]
    lib.mosh2_model_destroy.restype = None
    lib.mosh2_job_create.argtypes = [vp, C.POINTER(Options), C.c_int32, C.POINTER(Schedule), C.c_int32, C.POINTER(vp)]
    lib.mosh2_job_create_batch.argtypes = [vp, C.POINTER(Options), C.c_int32, _i32p, C.POINTER(Schedule), C.c_int32, C.POINTER(vp)]
    lib.mosh2_job_create_multi.argtypes = [C.POINTER(vp), C.c_int32, C.POINTER(Options), C.c_int32, _i32p, _i32p, C.POINTER(Schedule),
                                           C.c_int32, C.POINTER(vp)]
    lib.mosh2_job_upload.argtypes = [vp, _f64p, _u8p]
    lib.mosh2_job_linearize.argtypes = [vp, C.POINTER(Options), C.c_int32, C.c_int32, _f64p, C.POINTER(LinOut)]
    lib.mosh2_job_upload_markers.argtypes = [vp, _f64p, C.c_int32, C.c_int32, _i32p, C.c_int32, C.c_int32, C.c_double, _f64p]
    lib.mosh2_job_upload_markers_range.argtypes = [vp, C.c_int32, C.c_int32, _f64p, C.c_int32, C.c_int32, _i32p, C.c_int32, C.c_int32,
                                                   C.c_double, _f64p]
    lib.mosh2_job_upload_markers_folds.argtypes = [vp, C.c_int32, C.c_int32, _f64p, C.c_int32, C.c_int32, _i32p, _u8p, C.c_int32,
                                                   C.c_int32, C.c_double, _f64p]
    lib.mosh2_job_heldout_errors.argtypes = [vp, _f64p, _i32p]
    lib.mosh2_job_upload_device_range.argtypes = [vp, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp]
    lib.mosh2_job_upload_device.argtypes = [vp, vp, C.c_int32, vp, vp]
    lib.mosh2_job_row_width.argtypes = [vp]
    lib.mosh2_job_download_device.argtypes = [vp, vp]
    lib.mosh2_job_launch.argtypes = [vp]
    lib.mosh2_job_warm_states.argtypes = [vp, _f64p, _i32p]
    lib.mosh2_job_boundary_deltas.argtypes = [vp, C.c_int32, C.POINTER(C.c_float)]
    lib.mosh2_job_relaunch_chunks.argtypes = [vp, C.c_int32, _i32p, C.c_int32, C.c_int32, C.c_double, _i32p]
    lib.mosh2_job_sequence_sweep.argtypes = [vp, _f64p]
    lib.mosh2_job_download.argtypes = [vp, C.POINTER(Result)]
    lib.mosh2_job_sync.argtypes = [vp]
    lib.mosh2_job_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.mosh2_job_num_chunks.argtypes = [vp]
    lib.mosh2_job_chunk_ranges.argtypes = [vp, _i32p]
    lib.mosh2_job_span_ms.argtypes = [vp, vp, C.POINTER(C.c_float)]
    lib.mosh2_job_totals.argtypes = [vp, _i32p]
    lib.mosh2_job_destroy.argtypes = [vp]
    lib.mosh2_job_destroy.restype = None
    lib.mosh2_solve.argtypes = [vp, C.POINTER(Options), C.c_int32, _f64p, _u8p, C.POINTER(Schedule), C.c_int32,
                                C.POINTER(Result)]
    if path is None:
        _LIB = lib
    return lib


EXPORTED_SYMBOLS = (
    'mosh2_version', 'mosh2_last_error', 'mosh2_device_count', 'mosh2_default_options', 'mosh2_model_create',
    'mosh2_model_destroy', 'mosh2_job_create', 'mosh2_job_upload', 'mosh2_job_launch', 'mosh2_job_download',
    'mosh2_job_sync', 'mosh2_job_kernel_ms', 'mosh2_job_num_chunks', 'mosh2_job_totals', 'mosh2_job_destroy',
    'mosh2_solve', 'mosh2_job_upload_device', 'mosh2_job_row_width', 'mosh2_job_download_device', 'mosh2_job_span_ms',
    'mosh2_job_create_batch', 'mosh2_job_upload_device_range', 'mosh2_job_warm_states', 'mosh2_job_relaunch_chunks',
    'mosh2_job_boundary_deltas', 'mosh2_release_cached_memory', 'mosh2_mesh_distance', 'mosh2_job_upload_markers', 'mosh2_job_linearize',
    'mosh2_job_chunk_ranges', 'mosh2_job_upload_markers_range', 'mosh2_job_create_multi',
    'mosh2_job_sequence_sweep', 'mosh2_job_upload_markers_folds', 'mosh2_job_heldout_errors')


def _ptr(a: np.ndarray, typ):
    return a.ctypes.data_as(typ)


class DescHolder:
    """Keeps the contiguous arrays alive next to the ctypes struct that points into them."""

    def __init__(self, pk: StageIIPack):
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        self.arrays = dict(
            parents=i32(pk.parents), w_joint=i32(pk.w_joint),
            hand_comps=f64(pk.hand_comps), hands_mean=f64(pk.hands_mean), v0=f64(pk.v0), sd=f64(pk.sd), pd=f64(pk.pd),
            w_val=f64(pk.w_val), j0=f64(pk.j0), jd=f64(pk.jd), coefs=f64(pk.coefs),
            prior_means=f64(pk.prior_means), prior_Q=f64(pk.prior_Q), prior_neglogw=f64(pk.prior_neglogw),
            free1=i32(pk.free_step1), free2=i32(pk.free_step2))
        a = self.arrays
        d = ModelDesc()
        d.n_joints, d.n_markers, d.body_dof, d.p_red = pk.n_joints, pk.n_markers, pk.body_dof, pk.p_red
        d.n_hand_red, d.n_hand_full, d.n_dmpl = pk.n_hand_red, pk.n_hand_full, pk.n_dmpl
        d.kw = pk.kw
        for k in ('parents', 'w_joint', 'free1', 'free2'):
            setattr(d, k, _ptr(a[k], _i32p))
        for k in ('hand_comps', 'hands_mean', 'v0', 'sd', 'pd', 'w_val', 'j0', 'jd', 'coefs', 'prior_means',
                  'prior_Q', 'prior_neglogw'):
            setattr(d, k, _ptr(a[k], _f64p))
        d.prior_k, d.prior_d, d.prior_off = pk.prior_k, pk.prior_d, pk.prior_off
        if getattr(pk, 'prior_ids', None) is not None and len(pk.prior_ids):
            self.arrays['prior_ids'] = i32(pk.prior_ids)
            d.prior_ids = _ptr(self.arrays['prior_ids'], _i32p)
        d.n_free1, d.n_free2 = len(pk.free_step1), len(pk.free_step2)
        d.finger_lo, d.finger_hi = pk.finger_lo, pk.finger_hi
        d.n_expr, d.face_lo, d.face_hi = pk.n_expr, pk.face_lo, pk.face_hi
        jid = getattr(pk, 'jangles_ids', None)
        if jid is not None and len(jid):
            self.arrays['jangles_ids'], self.arrays['jangles_signs'] = i32(jid), f64(pk.jangles_signs)
            d.n_jangles = len(jid)
            d.jangles_ids, d.jangles_signs = _ptr(self.arrays['jangles_ids'], _i32p), _ptr(self.arrays['jangles_signs'], _f64p)
        self.desc = d


def make_options(weights=None, *, maxiter: int = 100, optimize_fingers: bool = False,
                 optimize_dynamics: bool = False, optimize_face: bool = False, robust_sigma: float = 0.0) -> Options:
    """Stage-II weights (moshpp_conf.yaml:118-125) -> mosh2_options.  ``robust_sigma`` > 0 (metres): the Geman-McClure
    data term (include/mosh2.h); 0: the reference's least squares."""
    o = Options(wt_data=400., wt_poseB=1.6, wt_poseH=1.0, wt_velo=2.5, wt_dmpl=1.0, wt_annealing=2.5,
                wt_extrap_dmpl=6.0, num_train_markers=46., delta_0=0.5, e3_first=1e-3, e3=1e-2, maxiter=maxiter,
                optimize_fingers=int(optimize_fingers), optimize_dynamics=int(optimize_dynamics),
                wt_poseF=1.0, wt_expr=1.0, optimize_face=int(optimize_face), robust_sigma=float(robust_sigma))
    if weights is not None:
        g = (lambda k: weights[k])
        o.wt_data, o.wt_poseB, o.wt_poseH = float(g('stageii_wt_data')), float(g('stageii_wt_poseB')), float(g('stageii_wt_poseH'))
        o.wt_velo, o.wt_dmpl = float(g('stageii_wt_velo')), float(g('stageii_wt_dmpl'))
        o.wt_annealing = float(g('stageii_wt_annealing'))
        for key, attr in (('stageii_wt_poseF', 'wt_poseF'), ('stageii_wt_expr', 'wt_expr')):
            try:
                setattr(o, attr, float(weights[key]))
            except (KeyError, AttributeError):
                pass
    return o


class ResultArrays:
    def __init__(self, n_frames: int, pk_dims: Dict[str, int]):
        F, M, nj, pr, nd = n_frames, pk_dims['M'], pk_dims['nJ'], pk_dims['p_red'], pk_dims['nd']
        self.fullpose = np.zeros((F, 3 * nj))
        self.pose = np.zeros((F, pr))
        self.trans = np.zeros((F, 3))
        self.dmpls = np.zeros((F, max(nd, 1)))
        self.markers_sim = np.zeros((F, M, 3))
        self.errs = np.zeros((F, len(ERR_NAMES)))
        self.status = np.zeros(F, dtype=np.int32)
        self.counters = np.zeros((F, 4), dtype=np.int32)
        self.nd = nd
        r = Result()
        r.fullpose, r.pose, r.trans = _ptr(self.fullpose, _f64p), _ptr(self.pose, _f64p), _ptr(self.trans, _f64p)
        r.dmpls = _ptr(self.dmpls, _f64p)
        r.markers_sim, r.errs = _ptr(self.markers_sim, _f64p), _ptr(self.errs, _f64p)
        r.status, r.counters = _ptr(self.status, _i32p), _ptr(self.counters, _i32p)
        self.c = r


def pack_dims(pk: StageIIPack) -> Dict[str, int]:
    return dict(M=pk.n_markers, nJ=pk.n_joints, p_red=pk.p_red, nd=pk.n_dmpl)


class Model:
    """Owns a ``mosh2_model`` handle on one GPU."""

    def __init__(self, pk: StageIIPack, device: int = 0, library_path: Optional[str] = None):
        self.lib = load_library(library_path)
        self.pk = pk
        self.holder = DescHolder(pk)
        self.handle = C.c_void_p()
        self.device = device
        rc = self.lib.mosh2_model_create(C.byref(self.holder.desc), device, C.byref(self.handle))
        if rc != 0:
            raise Mosh2Error(f'mosh2_model_create failed ({rc}): {self.lib.mosh2_last_error().decode()}')

    def _check(self, rc, what):
        if rc != 0:
            raise Mosh2Error(f'{what} failed ({rc}): {self.lib.mosh2_last_error().decode()}')

    def solve(self, obs: np.ndarray, vis: np.ndarray, options: Options, *, chunk_len: int = 0,
              chunk_warmup: int = 0, warmup_full: int = -1, precision: int = MOSH2_F32, first_extra: int = 0) -> ResultArrays:
        """One blocking call: H2D, kernel, D2H (mosh2_solve)."""
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        vis8 = np.ascontiguousarray(vis, dtype=np.uint8)
        F = obs.shape[0]
        assert obs.shape == (F, self.pk.n_markers, 3) and vis8.shape == (F, self.pk.n_markers)
        res = ResultArrays(F, pack_dims(self.pk))
        sched = make_schedule(chunk_len, chunk_warmup, warmup_full, first_extra)
        rc = self.lib.mosh2_solve(self.handle, C.byref(options), F, _ptr(obs, _f64p), _ptr(vis8, _u8p),
                                  C.byref(sched), precision, C.byref(res.c))
        self._check(rc, 'mosh2_solve')
        return res

    def job(self, n_frames: int, options: Options, *, chunk_len: int = 0, chunk_warmup: int = 0,
            warmup_full: int = -1, precision: int = MOSH2_F32, first_extra: int = 0) -> 'Job':
        """``n_frames``: frames of one sequence, or a list of frame counts = several sequences of this subject solved by
        one launch (mosh2_job_create_batch); the job's frame axis then holds them back to back."""
        return Job(self, n_frames, options, make_schedule(chunk_len, chunk_warmup, warmup_full, first_extra), precision)

    def close(self):
        if self.handle:
            self.lib.mosh2_model_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def multi_job(models, model_of_seq, counts, options: Options, *, chunk_len: int = 0, chunk_warmup: int = 0, warmup_full: int = -1,
              first_extra: int = 0, precision: int = MOSH2_F32) -> 'Job':
    """Sequences of several subjects solved by one launch (mosh2_job_create_multi): sequence q has ``counts[q]`` frames and is
    solved with ``models[model_of_seq[q]]``.  The models (``Model``, one device, one kernel shape) must stay open while the job
    lives.  Returns a ``Job`` with the interface of a batch job; its frame axis holds the sequences back to back."""
    return Job(models[0], counts, options, make_schedule(chunk_len, chunk_warmup, warmup_full, first_extra), precision,
               models=list(models), model_of_seq=model_of_seq)


class Job:
    """Staged upload / launch / download on device-resident buffers (used by bench.py)."""

    def __init__(self, model: Model, n_frames, options: Options, schedule: Schedule, precision: int, *, models=None,
                 model_of_seq=None):
        counts = np.ascontiguousarray(np.atleast_1d(n_frames), dtype=np.int32)
        self.frame_counts = counts
        self.seq_offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        n_frames = int(counts.sum())
        self.model, self.lib, self.n_frames = model, model.lib, n_frames
        self.handle = C.c_void_p()
        self.options = options
        self.schedule = schedule
        self.models = models            # multi-model job: every model, kept referenced while the job lives
        if models is None:
            rc = self.lib.mosh2_job_create_batch(model.handle, C.byref(options), len(counts), _ptr(counts, _i32p), C.byref(schedule),
                                                 precision, C.byref(self.handle))
            model._check(rc, 'mosh2_job_create')
        else:
            mos = np.ascontiguousarray(model_of_seq, dtype=np.int32)
            if mos.shape != counts.shape:
                raise ValueError(f'{len(counts)} sequences, {len(mos)} model indices')
            handles = (C.c_void_p * len(models))(*[m.handle for m in models])
            rc = self.lib.mosh2_job_create_multi(handles, len(models), C.byref(options), len(counts), _ptr(counts, _i32p), _ptr(mos, _i32p),
                                                 C.byref(schedule), precision, C.byref(self.handle))
            model._check(rc, 'mosh2_job_create_multi')
        self.result = ResultArrays(n_frames, pack_dims(model.pk))

    def upload(self, obs: np.ndarray, vis: np.ndarray):
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        vis8 = np.ascontiguousarray(vis, dtype=np.uint8)
        self.model._check(self.lib.mosh2_job_upload(self.handle, _ptr(obs, _f64p), _ptr(vis8, _u8p)), 'mosh2_job_upload')

    def upload_markers(self, raw: np.ndarray, col_of_marker, frame_start: int, frame_step: int, unit_per_metre: float, rot3x3=None):
        """The mocap input adapter on the device over the whole frame axis (``upload_markers_range`` from frame 0, as
        mosh2_job_upload_markers does): ``raw`` = the capture file's marker table
        [file frames, file columns, 3] float64 in file units; ``col_of_marker[i]`` = file column of latent marker i (-1: absent);
        job frame f = file frame frame_start + f * frame_step."""
        self.upload_markers_range(0, self.n_frames, raw, col_of_marker, frame_start, frame_step, unit_per_metre, rot3x3)

    def upload_markers_range(self, frame0: int, n: int, raw: np.ndarray, col_of_marker, frame_start: int, frame_step: int,
                             unit_per_metre: float, rot3x3=None):
        """``upload_markers`` for frames [frame0, frame0 + n) of the job's frame axis: one capture of a batch job
        (mosh2_job_upload_markers_range).  The library stages the rows it needs before it returns, so the uploads of all
        captures can be issued back to back."""
        raw = np.ascontiguousarray(raw, dtype=np.float64)
        cols = np.ascontiguousarray(col_of_marker, dtype=np.int32)
        assert raw.ndim == 3 and raw.shape[2] == 3 and cols.shape == (self.model.pk.n_markers,)
        rot = None if rot3x3 is None else np.ascontiguousarray(rot3x3, dtype=np.float64).reshape(3, 3)
        self.model._check(self.lib.mosh2_job_upload_markers_range(self.handle, int(frame0), int(n), _ptr(raw, _f64p), raw.shape[0],
                                                                  raw.shape[1], _ptr(cols, _i32p), int(frame_start), int(frame_step),
                                                                  float(unit_per_metre), _ptr(rot, _f64p) if rot is not None else None),
                          'mosh2_job_upload_markers_range')

    def upload_markers_folds(self, seq0: int, hide, raw: np.ndarray, col_of_marker, frame_start: int, frame_step: int,
                             unit_per_metre: float, rot3x3=None):
        """Held-out folds of one capture (mosh2_job_upload_markers_folds): sequence seq0 + k of the job is the capture with the
        markers ``hide[k]`` ([n_folds, M] bool) deleted; the other arguments as in ``upload_markers_range``.  The raw table is
        staged once for all folds."""
        raw = np.ascontiguousarray(raw, dtype=np.float64)
        cols = np.ascontiguousarray(col_of_marker, dtype=np.int32)
        h = np.ascontiguousarray(hide, dtype=np.uint8)
        assert raw.ndim == 3 and raw.shape[2] == 3 and cols.shape == (self.model.pk.n_markers,)
        assert h.ndim == 2 and h.shape[1] == self.model.pk.n_markers
        rot = None if rot3x3 is None else np.ascontiguousarray(rot3x3, dtype=np.float64).reshape(3, 3)
        self.model._check(self.lib.mosh2_job_upload_markers_folds(self.handle, int(seq0), h.shape[0], _ptr(raw, _f64p), raw.shape[0],
                                                                  raw.shape[1], _ptr(cols, _i32p), _ptr(h, _u8p), int(frame_start),
                                                                  int(frame_step), float(unit_per_metre),
                                                                  _ptr(rot, _f64p) if rot is not None else None),
                          'mosh2_job_upload_markers_folds')
        self.folds = (int(seq0), h.shape[0], int(h.sum(1).max()))

    def heldout_errors(self):
        """(err [n_folds, n, K], status [n_folds, n]) of the last ``upload_markers_folds``, computed on the device from the job's
        current rows (mosh2_job_heldout_errors): the error in metres of the r-th marker fold k hides in frame t, NaN where undefined."""
        seq0, n_folds, K = self.folds
        n = int(self.frame_counts[seq0])
        err = np.zeros((n_folds, n, K))
        st = np.zeros((n_folds, n), dtype=np.int32)
        self.model._check(self.lib.mosh2_job_heldout_errors(self.handle, _ptr(err, _f64p), _ptr(st, _i32p)), 'mosh2_job_heldout_errors')
        return err, st

    def linearize(self, x: np.ndarray, options: Options, step: int, build: bool) -> Dict[str, np.ndarray]:
        """mosh2_job_linearize: every frame of the job evaluated (and, with ``build``, linearised) at its row of ``x``
        [F, 3 + p_red + n_dmpl]; see include/mosh2.h.  Needs a job of one-frame chunks and uploaded observations.  A float32
        job evaluates at ``x`` rounded to float32 and returns its float32 results as float64 arrays."""
        pk = self.model.pk
        F, M = self.n_frames, pk.n_markers
        n = len(pk.free_step2) if step == 2 else len(pk.free_step1)
        x = np.ascontiguousarray(x, dtype=np.float64)
        assert x.shape == (F, pk.nx)
        out = dict(errs=np.zeros((F, len(ERR_NAMES))), markers_sim=np.zeros((F, M, 3)), r=np.zeros((F, 3 * M)), vp=np.zeros((F, 3 * M, 3)))
        if build:
            out.update(A=np.zeros((F, n, n)), g=np.zeros((F, n)), J=np.zeros((F, 3 * M, n)))
        c = LinOut(*[_ptr(out[k], _f64p) if k in out else None for k in ('errs', 'markers_sim', 'r', 'vp', 'A', 'g', 'J')])
        self.model._check(self.lib.mosh2_job_linearize(self.handle, C.byref(options), int(step), int(bool(build)), _ptr(x, _f64p),
                                                       C.byref(c)), 'mosh2_job_linearize')
        return out

    def upload_device(self, d_obs_ptr: int, obs_is_f64: bool, d_vis_ptr: int, producer_stream: int = 0):
        """Observations already on this job's GPU (raw device pointers, e.g. ``tensor.data_ptr()`` of an NCCL receive
        buffer; ``producer_stream`` = the cudaStream_t the producer was queued on)."""
        self.model._check(self.lib.mosh2_job_upload_device(self.handle, C.c_void_p(d_obs_ptr), int(bool(obs_is_f64)),
                                                           C.c_void_p(d_vis_ptr), C.c_void_p(producer_stream)),
                          'mosh2_job_upload_device')

    def upload_device_range(self, frame0: int, n: int, d_obs_ptr: int, obs_is_f64: bool, d_vis_ptr: int, producer_stream: int = 0):
        """... for frames [frame0, frame0 + n) of the job's frame axis (one sequence of a batch job)."""
        self.model._check(self.lib.mosh2_job_upload_device_range(self.handle, int(frame0), int(n), C.c_void_p(d_obs_ptr),
                                                                 int(bool(obs_is_f64)), C.c_void_p(d_vis_ptr),
                                                                 C.c_void_p(producer_stream)), 'mosh2_job_upload_device_range')

    @property
    def row_width(self) -> int:
        return int(self.lib.mosh2_job_row_width(self.handle))

    def download_device(self, d_rows_ptr: int):
        """Packed float32 result rows into a device buffer of n_frames * row_width floats (include/mosh2.h)."""
        self.model._check(self.lib.mosh2_job_download_device(self.handle, C.c_void_p(d_rows_ptr)), 'mosh2_job_download_device')

    def launch(self):
        self.model._check(self.lib.mosh2_job_launch(self.handle), 'mosh2_job_launch')

    def sync(self):
        self.model._check(self.lib.mosh2_job_sync(self.handle), 'mosh2_job_sync')

    def warm_states(self):
        """(x [n_chunks, 3 + p_red + n_dmpl], frame [n_chunks]): the state every chunk reached on its last warm-up frame and
        that frame's index (-1: the chunk starts its sequence).  See mosh2_job_warm_states."""
        pk = self.model.pk
        n = self.num_chunks
        x = np.zeros((n, 3 + pk.p_red + pk.n_dmpl))
        fr = np.zeros(n, dtype=np.int32)
        self.model._check(self.lib.mosh2_job_warm_states(self.handle, _ptr(x, _f64p), _ptr(fr, _i32p)), 'mosh2_job_warm_states')
        return x, fr

    def boundary_deltas(self):
        """Per chunk: max |warm-up state - emitted result| on the chunk's last warm-up frame, split into
        (root + body pose [rad], remaining pose coefficients, translation [m], dmpl / expression coefficients);
        computed on the device from the last launch (mosh2_job_boundary_deltas)."""
        pk = self.model.pk
        out = np.zeros((self.num_chunks, 4), dtype=np.float32)
        self.model._check(self.lib.mosh2_job_boundary_deltas(self.handle, min(pk.body_dof, 66), out.ctypes.data_as(C.POINTER(C.c_float))),
                          'mosh2_job_boundary_deltas')
        return out.astype(np.float64)

    def relaunch_chunks(self, chunk_ids, chunk_warmup: int, warmup_full: int = -1, merge_tol: float = 0.0, root_turns=None):
        """Re-solves the listed chunks; ``chunk_warmup < 0`` = resume from the emitted rows; ``root_turns``: per listed chunk,
        full turns added to the root angle of its cold start (mosh2_job_relaunch_chunks)."""
        ids = np.ascontiguousarray(chunk_ids, dtype=np.int32)
        turns = None if root_turns is None else np.ascontiguousarray(root_turns, dtype=np.int32)
        if turns is not None and turns.shape != ids.shape:
            raise ValueError('root_turns: one value per chunk')
        self.model._check(self.lib.mosh2_job_relaunch_chunks(self.handle, len(ids), _ptr(ids, _i32p), int(chunk_warmup),
                                                             int(warmup_full), float(merge_tol),
                                                             None if turns is None else _ptr(turns, _i32p)),
                          'mosh2_job_relaunch_chunks')

    def sequence_sweep(self) -> np.ndarray:
        """One sweep of the joint minimisation of the sequence objective over the job's rows (mosh2_job_sequence_sweep); returns
        the largest change of any processed frame's row, per group as in ``boundary_deltas``."""
        out = np.zeros(4)
        self.model._check(self.lib.mosh2_job_sequence_sweep(self.handle, _ptr(out, _f64p)), 'mosh2_job_sequence_sweep')
        return out

    def download(self) -> ResultArrays:
        self.model._check(self.lib.mosh2_job_download(self.handle, C.byref(self.result.c)), 'mosh2_job_download')
        return self.result

    def kernel_ms(self) -> float:
        ms = C.c_float()
        self.model._check(self.lib.mosh2_job_kernel_ms(self.handle, C.byref(ms)), 'mosh2_job_kernel_ms')
        return float(ms.value)

    def span_ms(self, last: 'Job') -> float:
        """Device time from the start of this job's last launch to the end of ``last``'s (same device)."""
        ms = C.c_float()
        self.model._check(self.lib.mosh2_job_span_ms(self.handle, last.handle, C.byref(ms)), 'mosh2_job_span_ms')
        return float(ms.value)

    def totals(self) -> Dict[str, int]:
        """Work of the last launch over all processed frames (warm-up included) and over the emitted frames only."""
        t = np.zeros(8, dtype=np.int32)
        self.model._check(self.lib.mosh2_job_totals(self.handle, _ptr(t, _i32p)), 'mosh2_job_totals')
        return dict(iterations=int(t[0]), evaluations=int(t[1]), builds=int(t[2]), minimisations=int(t[3]),
                    emitted_iterations=int(t[4]), emitted_evaluations=int(t[5]), emitted_builds=int(t[6]),
                    emitted_minimisations=int(t[7]))

    @property
    def num_chunks(self) -> int:
        return int(self.lib.mosh2_job_num_chunks(self.handle))

    def chunk_ranges(self) -> np.ndarray:
        """[n_chunks, 2]: first emitted frame and end of the emitted range of every chunk (job frame axis)."""
        out = np.zeros((self.num_chunks, 2), dtype=np.int32)
        self.model._check(self.lib.mosh2_job_chunk_ranges(self.handle, _ptr(out, _i32p)), 'mosh2_job_chunk_ranges')
        return out

    def close(self):
        if self.handle:
            self.lib.mosh2_job_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
