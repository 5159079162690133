"""``mosh_stageii`` -- drop-in for the reference's Stage-II callable, running on libmosh2.so (H100).

Reference: src/moshpp/chmosh.py:458-741.  Same positional signature, same return dictionary
(chmosh.py:726-741), same frame-skip rule (586-588); it plugs into the reference's own call site
``MoSh.mosh_stageii(mosh_stageii_func)`` (mosh_head.py:268-301) unchanged:

    from moshpp_b200.chmosh import mosh_stageii
    mp.mosh_stageii(mosh_stageii)

What runs where
  host (this file, pack.py, mocap_interface.py): file IO, label matching, once-per-subject packing;
  device (csrc/): every per-frame evaluation -- SMPL forward, Jacobians, priors, normal equations,
  Cholesky, dog-leg, the frame loop itself.  There is no CPU solver: without libmosh2.so or a GPU the
  call raises.

Parallel-in-time schedule (DESIGN.md section 4): the frames are cut into chunks solved concurrently,
each started ``chunk_warmup`` frames early.  The reference's recursion is contractive, so the chunked
result converges geometrically in the warm-up length to the sequential one (measured on C2: 1.5e-4 rad /
0.03 mm in the simulated markers at the default 48 frames, 1.3e-5 rad / 0.006 mm at 64; DESIGN.md section 4);
``chunk_len=0`` runs the reference's single sequential pass exactly.
"""
from __future__ import annotations

import hashlib
import logging
import math
import os
import time
from collections import OrderedDict
from typing import Optional

import numpy as np

from . import lib as _lib
from . import pack as _pack
from .mocap_interface import MocapSession, rotation_xyz as _rotation_xyz

logger = logging.getLogger('moshpp_b200')

NUM_SMS = 132                # H100 SXM: thread blocks of the Stage-II kernel that run at once (one per SM)
DEFAULT_WARMUP = 64          # solved frames every chunk is started early (DESIGN.md section 4)
DEFAULT_WARMUP_FULL = 48     # the last 48 of them with the full per-frame schedule, the first 16 with one Step-2 iteration


def _get(node, key, default=None):
    try:
        return node[key]
    except (KeyError, TypeError, IndexError):
        return getattr(node, key, default)


def _read_vertices(fname: str) -> np.ndarray:
    """v_template file (the reference uses psbody.mesh.Mesh, smpl_fast_derivatives.py:73-78)."""
    if fname.endswith('.npy'):
        return np.load(fname)
    if fname.endswith('.obj'):
        return np.array([[float(x) for x in l.split()[1:4]] for l in open(fname) if l.startswith('v ')])
    if fname.endswith('.ply'):
        with open(fname, 'rb') as f:
            header = []
            while True:
                line = f.readline().decode('latin-1').strip()
                header.append(line)
                if line == 'end_header':
                    break
            n = int([h for h in header if h.startswith('element vertex')][0].split()[-1])
            nprops = 0
            in_vertex = False
            for h in header:
                if h.startswith('element'):
                    in_vertex = h.startswith('element vertex')
                elif h.startswith('property') and in_vertex:
                    nprops += 1
            if any('ascii' in h for h in header):
                return np.array([[float(x) for x in f.readline().split()[:3]] for _ in range(n)])
            if any('binary_little_endian' in h for h in header) and all(
                    h.split()[1] == 'float' for h in header if h.startswith('property') and 'list' not in h):
                return np.frombuffer(f.read(4 * nprops * n), dtype='<f4').reshape(n, nprops)[:, :3].astype(np.float64)
    raise NotImplementedError(f'cannot read v_template from {fname}')


def first_chunk_extra(warmup: int = DEFAULT_WARMUP, warmup_full: int = DEFAULT_WARMUP_FULL) -> int:
    """mosh2_schedule.first_extra of the planned schedules: what a warm-up costs in fully solved frames (light frames count
    a quarter).  The first chunk of a sequence has no warm-up; emitting that many frames more it finishes with the others."""
    wf = warmup if (warmup_full < 0 or warmup_full > warmup) else warmup_full
    return int(wf + (warmup - wf) // 4) if warmup > 0 else 0


def count_chunks(n_frames: int, chunk_len: int, first_extra: int = 0) -> int:
    """Chunks mosh2_host::chunk_table cuts a sequence of ``n_frames`` into."""
    if chunk_len <= 0 or chunk_len >= n_frames:
        return 1
    if first_extra > 0:
        rest = n_frames - chunk_len - first_extra
        return 1 + (-(-rest // chunk_len) if rest > 0 else 0)
    return -(-n_frames // chunk_len)


def plan_chunk_len(frame_counts, sm_budget: int = NUM_SMS, warmup: int = DEFAULT_WARMUP,
                   warmup_full: int = DEFAULT_WARMUP_FULL, min_len: int = 4, first_extra: int = 0) -> int:
    """Chunk length for a set of sequences that are solved together on one GPU (one thread block per chunk, one block
    per SM at a time).  The chunks run in waves of ``sm_budget``; a wave lasts as long as its longest chunk, i.e. about
    chunk_len + warm-up frame solves.  Returns the length that minimises waves x (chunk_len + warm-up cost), where the
    light warm-up frames cost about a quarter of a full one and the cold start about five.  ``first_extra``: frames the
    first chunk of every sequence emits on top (``first_chunk_extra``)."""
    counts = [int(f) for f in frame_counts if f > 0]
    if not counts:
        return min_len
    w_cost = warmup_full + 0.25 * max(0, warmup - warmup_full) + 5.0
    best = None
    for waves in range(1, 9):
        lo, hi = min_len, max(max(counts), min_len)
        while lo < hi:                                   # smallest L whose chunks fit `waves` waves
            mid = (lo + hi) // 2
            if sum(count_chunks(f, mid, first_extra) for f in counts) <= waves * sm_budget:
                hi = mid
            else:
                lo = mid + 1
        cost = waves * (lo + w_cost)
        if best is None or cost < best[0] - 1e-9:
            best = (cost, lo)
        if lo == min_len:
            break
    return best[1]


def auto_chunk_len(n_frames: int, sm_budget: int = NUM_SMS) -> int:
    """Shortest chunks that still give about one chunk per available SM (latency = chunk_len + warm-up)."""
    return max(4, int(math.ceil(n_frames / max(1, sm_budget))))


# ---------------------------------------------------------------------------------------------------------------------
# Subject cache.  Everything ``prepare_stageii`` computes -- and the device copy of it -- depends on the subject (body
# model file, shape, latent markers, layout, options), not on the sequence; a subject usually comes with many sequences
# (the reference re-does this work per call).  The packed constants and their device model are kept for the last few
# subjects, keyed by the CONTENT of every input (file identity = path + mtime + size).  Nothing sequence-dependent is cached.
# ---------------------------------------------------------------------------------------------------------------------
_SUBJECT_CACHE: 'OrderedDict[tuple, dict]' = OrderedDict()
SUBJECT_CACHE_SIZE = 4


def _file_id(fname):
    if not fname:
        return None
    try:
        st = os.stat(str(fname))
        return (os.path.realpath(str(fname)), st.st_mtime_ns, st.st_size)
    except OSError:
        return (str(fname), None, None)


def _subject_key(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device):
    sm, mp = cfg.surface_model, cfg.moshpp
    h = hashlib.blake2b(digest_size=16)
    h.update(np.ascontiguousarray(betas, dtype=np.float64).tobytes())
    h.update(np.ascontiguousarray(markers_latent, dtype=np.float64).tobytes())
    w = cfg.opt_settings.weights
    scalars = (
        _file_id(sm.fname), _file_id(_get(mp, 'pose_hand_prior_fname')), _file_id(_get(mp, 'pose_body_prior_fname')),
        _file_id(_get(sm, 'dmpl_fname')) if _get(mp, 'optimize_dynamics', False) else None, _file_id(v_template_fname),
        str(sm.type), int(sm.num_betas), int(_get(sm, 'num_dmpls', 0) or 0), bool(sm.use_hands_mean), int(sm.dof_per_hand),
        int(_get(sm, 'betas_expr_start_id', 0) or 0), int(_get(sm, 'num_expressions', 0) or 0),
        bool(_get(mp, 'optimize_fingers', False)), bool(_get(mp, 'optimize_face', False)), bool(_get(mp, 'optimize_dynamics', False)),
        bool(_get(mp, 'optimize_toes', False)), int(cfg.opt_settings.maxiter),
        tuple(sorted((str(k), float(w[k])) for k in w.keys() if str(k).startswith('stageii_'))),
        tuple(latent_labels), tuple(marker_meta['marker_type_mask'].keys()), tuple(marker_meta['marker_type'].items()), int(device))
    h.update(repr(scalars).encode())
    return h.hexdigest()


def clear_subject_cache():
    while _SUBJECT_CACHE:
        _, e = _SUBJECT_CACHE.popitem(last=False)
        e['model'].close()


def subject_for(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None, device: int = 0):
    """(StageIIPack, options, flags, lib.Model on ``device``) of a subject, from the cache or freshly prepared."""
    key = _subject_key(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device)
    e = _SUBJECT_CACHE.get(key)
    if e is None:
        pk, opts, flags = prepare_stageii(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname)
        e = dict(pk=pk, opts=opts, flags=flags, model=_lib.Model(pk, device=device), hit=False)
        _SUBJECT_CACHE[key] = e
        while len(_SUBJECT_CACHE) > SUBJECT_CACHE_SIZE:
            _, old = _SUBJECT_CACHE.popitem(last=False)
            old['model'].close()
    else:
        _SUBJECT_CACHE.move_to_end(key)
        e['hit'] = True
        for k in ('optimize_fingers', 'optimize_face'):          # the gating side effect of prepare_stageii (chmosh.py:475-486)
            if not e['flags'][k] and bool(_get(cfg.moshpp, k, False)):
                try:
                    cfg.moshpp[k] = False
                except Exception:
                    pass
    return e['pk'], e['opts'], dict(e['flags']), e['model'], e['hit']


def prepare_stageii(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None):
    """Everything chmosh.py:475-514,548-579 does before the frame loop -> (StageIIPack, options, flags)."""
    sm, mp = cfg.surface_model, cfg.moshpp
    latent_labels = list(latent_labels)
    flags = {}
    for body_part, key in {'finger': 'optimize_fingers', 'face': 'optimize_face'}.items():       # chmosh.py:475-486
        on = bool(_get(mp, key, False))
        if on:
            if not np.any([body_part in m for m in marker_meta['marker_type_mask'].keys()]):
                logger.warning(f'{key} was activated but no {body_part} marker type detected in the marker layout')
                on = False
            elif not np.any([(body_part in t) and l in latent_labels for l, t in marker_meta['marker_type'].items()]):
                logger.warning(f'{key} was activated but no {body_part} marker type detected in the mocaps')
                on = False
            if not on:
                try:
                    mp[key] = False
                except Exception:
                    pass
        flags[key] = on
    if flags['optimize_face'] and sm.type != 'smplx':
        flags['optimize_face'] = False          # only SMPL-X has face pose ids / expression components (chmosh.py:560-566)

    v_template = _read_vertices(v_template_fname) if v_template_fname else None
    model = _pack.load_surface_model(sm.fname, pose_hand_prior_fname=_get(mp, 'pose_hand_prior_fname'),
                                     use_hands_mean=bool(sm.use_hands_mean), dof_per_hand=int(sm.dof_per_hand),
                                     v_template=v_template, surface_model_type=sm.type)
    if model.model_type != sm.type:
        raise ValueError(f'{model.model_type} != {sm.type}')                                       # bodymodel_loader.py:108
    prior = None
    prior_fname = _get(mp, 'pose_body_prior_fname')
    if prior_fname and model.model_type == 'animal_horse':
        prior = _pack.create_horse_body_prior(prior_fname)                                         # bodymodel_loader.py:121-125
    elif prior_fname and model.model_type != 'mano':
        prior = _pack.create_gmm_body_prior(prior_fname, exclude_hands=model.model_type in ('smplh', 'smplx'))
    dyn = bool(_get(mp, 'optimize_dynamics', False))
    dmpl_dirs = None
    if dyn:                                                                                        # chmosh.py:507-514
        if sm.type not in ('smpl', 'smplh'):
            logger.warning('DMPL with %s is rejected by the reference (chmosh.py:508-509); running the '
                           'extension defined in DESIGN.md', sm.type)
        dmpl_dirs = np.asarray(_pack.load_reference_pickle(sm.dmpl_fname)['eigvec'])
    pk = _pack.build_pack(model, np.asarray(betas, dtype=np.float64), np.asarray(markers_latent, dtype=np.float64),
                          num_betas=int(sm.num_betas), prior=prior, dmpl_dirs=dmpl_dirs,
                          num_dmpls=int(sm.num_dmpls) if dyn else 0,
                          optimize_fingers=flags['optimize_fingers'],
                          optimize_toes=bool(_get(mp, 'optimize_toes', False)),
                          optimize_face=flags['optimize_face'],
                          expr_start=int(_get(sm, 'betas_expr_start_id', 0) or 0),
                          num_expressions=int(_get(sm, 'num_expressions', 0) or 0) if flags['optimize_face'] else 0)
    flags['n_betas_model'] = int(model.shapedirs.shape[-1])
    flags['expr_start'] = int(_get(sm, 'betas_expr_start_id', 0) or 0)
    opts = _lib.make_options(cfg.opt_settings.weights, maxiter=int(cfg.opt_settings.maxiter),
                             optimize_fingers=flags['optimize_fingers'] and pk.finger_hi > pk.finger_lo,
                             optimize_dynamics=dyn, optimize_face=flags['optimize_face'] and pk.n_expr > 0)
    return pk, opts, flags


def observation_lists(obs: np.ndarray, vis: np.ndarray, latent_labels) -> dict:
    """The result-independent half of chmosh.py:712-718: per-frame lists of the observed markers and their labels over the
    frames with at least one visible marker (the frames the reference solves, chmosh.py:586-588).  Computed on the host
    while the device solves (``mosh_stageii``); ``assemble_stageii_data`` builds it itself when it is not handed over."""
    fid = np.nonzero(vis.any(1))[0]
    vf = vis if len(fid) == len(vis) else vis[fid]
    cnt = vf.sum(1)
    ends = np.cumsum(cnt)
    starts = ends - cnt
    # positions of the visible markers of the solved frames in the flattened (frame, marker) grid: one take() per array
    # (a fancy-index copy followed by a boolean gather costs ten times as much)
    M = vis.shape[1]
    flat_idx = np.flatnonzero(vf)
    if len(fid) != len(vis):
        flat_idx = flat_idx + (fid[flat_idx // M] - flat_idx // M) * M
    obs_cat = np.take(obs.reshape(-1, 3), flat_idx, axis=0)
    labels = np.asarray(latent_labels, dtype=object)
    # the label lists are built once per visibility pattern (drop-outs come in runs) and copied
    by_pattern: dict = {}
    labels_obs = []
    for row in vf:
        key = row.tobytes()
        names = by_pattern.get(key)
        if names is None:
            names = by_pattern[key] = labels[row].tolist()
        labels_obs.append(list(names))
    return {'fid': fid, 'vf': vf, 'starts': starts, 'ends': ends, 'flat_idx': flat_idx, 'labels_obs': labels_obs,
            'markers_obs': [obs_cat[a:b] for a, b in zip(starts, ends)]}


def assemble_stageii_data(res: '_lib.ResultArrays', obs: np.ndarray, vis: np.ndarray, latent_labels, pk,
                          flags, dyn: bool, lists: Optional[dict] = None) -> dict:
    """chmosh.py:712-741: per-frame lists over the frames that had at least one visible marker."""
    solved = (res.status & _lib.ST_SOLVED) != 0
    fid = np.nonzero(solved)[0]
    if lists is None or not np.array_equal(lists['fid'], fid):
        lists = observation_lists(obs, np.logical_and(vis, solved[:, None]), latent_labels)
    st = res.status[fid]
    errs = {'data': res.errs[fid, 0]}
    if pk.prior_k:
        errs['poseB'] = res.errs[fid, 1]
    if len(getattr(pk, 'jangles_ids', ())):
        errs['poseB_jangles'] = res.errs[fid, 3]       # (animal_horse: the finger column carries the joint-angle term)
    if flags['optimize_fingers'] and pk.finger_hi > pk.finger_lo:
        errs['poseH'] = res.errs[fid, 3]
    face = bool(flags.get('optimize_face')) and pk.n_expr > 0
    if face:
        errs['poseF'] = res.errs[fid, 6]
        errs['expr'] = res.errs[fid, 7]
    if dyn:
        errs['dmpl'] = res.errs[fid, 4]
        errs['extrap_dmpl'] = res.errs[fid, 5][(st & _lib.ST_HAS_EXTRAP) != 0]
    errs['velo'] = res.errs[fid, 2][(st & _lib.ST_HAS_VELO) != 0]
    errs = {k: np.array(v) for k, v in errs.items() if k in ('data', 'poseB', 'poseB_jangles', 'poseH', 'dmpl', 'poseF', 'expr') or len(v)}
    every = len(fid) == len(res.status)          # (the result arrays belong to this call: no second copy)
    data = {
        'fullpose': res.fullpose if every else res.fullpose[fid],
        'trans': res.trans if every else res.trans[fid],
    }
    if dyn:
        data['dmpls'] = res.dmpls[fid, :pk.n_dmpl - pk.n_expr].copy()
    if face:
        # chmosh.py:724 stores betas[exp_start:], i.e. the optimised coefficients followed by the model's remaining
        # (untouched, zero) shape components
        tail = max(pk.n_expr, int(flags.get('n_betas_model', 0)) - int(flags.get('expr_start', 0)))
        expr = np.zeros((len(fid), tail))
        expr[:, :pk.n_expr] = res.dmpls[fid, pk.n_dmpl - pk.n_expr:pk.n_dmpl]
        data['expression'] = expr
    # per-frame lists over the visible markers (chmosh.py:716-718): one gather, cut into per-frame views
    sim_cat = np.take(res.markers_sim.reshape(-1, 3), lists['flat_idx'], axis=0)
    data['stageii_debug_details'] = {
        'stageii_errs': errs,
        'markers_sim': [sim_cat[a:b] for a, b in zip(lists['starts'], lists['ends'])],
        'markers_obs': lists['markers_obs'],
        'labels_obs': lists['labels_obs'],
    }
    return data


# Boundary tolerances of the chunked schedule: what a chunk's warm-up state may differ from the emitted result of the same
# frame (root+body pose rad, other pose coefficients, translation m, dmpl / expression coefficients).  'fast' keeps the
# chunk starts a factor of three inside BASELINE.md section 4's per-frame tolerances; 'exact' is the parity mode.
BOUNDARY_TOL = {'fast': (3e-4, 3e-3, 3e-5, 3e-3), 'exact': (1e-6, 1e-5, 1e-7, 1e-5)}


def default_schedule(model_type: str, mode: str = 'fast', n_linear: int = 0):
    """The schedule a sequence is solved with by default; ``solve_verified`` repairs the chunk boundaries the warm-up left
    open.  The reference's frame recursion forgets its start geometrically, at a rate set by the
    velocity term against the weakest other term on a pose coefficient (DESIGN.md section 4): 0.86 per frame for the
    body models, 0.93 for the hand-only MANO model (no body prior: only poseH holds the finger coefficients).

    The fast preset (float32, 64/48, boundary tolerance a third of the per-frame tolerance) is the default only where it
    follows the reference's float64 trajectory on >= 99 % of the frames (measured, DESIGN.md section 5): SMPL / SMPL-H /
    SMPL-X without per-frame linear coefficients.  With DMPL or expression coefficients (``n_linear`` > 0) the frame
    objective has more nearly flat directions and, on BASELINE config 3, a second self-consistent branch that cold starts
    fall into: 2-7 % of the frames left the tolerance under every fast schedule tried, in float32 and in float64.  Those
    models, and MANO in ``exact`` mode, run the exact preset (float64, 256 fully solved warm-up frames, tight boundary
    check); MANO's fast preset is float64 with a 256/224 warm-up (30 unknowns, no prior: a float32 cold start can take
    another branch of the dog-leg; 0.93 per frame).  Returns (chunk_warmup, warmup_full, precision, boundary tolerance)."""
    if mode == 'exact' or n_linear > 0:
        return 256, -1, 'f64', BOUNDARY_TOL['exact']
    if model_type == 'mano':
        return 256, 224, 'f64', BOUNDARY_TOL['fast']
    return DEFAULT_WARMUP, DEFAULT_WARMUP_FULL, 'f32', BOUNDARY_TOL['fast']


# A chunk whose warm-up state differs from the emitted row by more than this (rad, root + body pose) may have started on
# another axis-angle branch of the root: two branches of one rotation lie 2 pi / sqrt(3) > 3.6 rad apart in some component,
# the boundary deltas of a converged warm-up are below 1e-3.
ROOT_BRANCH_DELTA = 1.0


def root_branch_turns(root: np.ndarray, solved: np.ndarray, ranges: np.ndarray, seq_starts) -> np.ndarray:
    """Full turns that put every chunk on the root branch of the sequential pass.

    The sequential pass aligns the first frame of a sequence (angle in [0, pi]) and then tracks the root as a free
    parameter: once the body has turned past pi, its axis-angle root lies beyond pi.  A chunk aligns the first frame of its
    own warm-up and so starts on the principal branch: behind such a crossing it tracks u (theta - 2 pi n) where the
    sequential pass tracks u theta.  This pass walks the chunks of every sequence in order and unwraps the emitted root across
    each chunk boundary -- the first solved root of a chunk onto the equivalent rotation vector u (theta + 2 pi n) nearest to
    the (unwrapped) last solved root in front of it.  ``root`` [F, 3] emitted roots, ``solved`` [F] bool, ``ranges``
    [n_chunks, 2] emitted ranges (``Job.chunk_ranges``), ``seq_starts``: first frames of the sequences.  Returns n per chunk
    (0: the chunk is on the branch of the chunks in front of it)."""
    starts = set(int(s) for s in seq_starts)
    turns = np.zeros(len(ranges), dtype=np.int64)
    last = None                                   # unwrapped last solved root in front of the chunk
    for c, (a, b) in enumerate(ranges):
        if int(a) in starts:
            last = None
        fs = np.flatnonzero(solved[a:b]) + a
        if not len(fs):
            continue
        r0, r1 = root[fs[0]], root[fs[-1]]
        if last is not None:
            th = np.linalg.norm(r0)
            if th > 0:
                turns[c] = int(np.round((r0 @ last / th - th) / (2 * np.pi)))
        th1 = np.linalg.norm(r1)
        last = r1 * (1 + 2 * np.pi * turns[c] / th1) if th1 > 0 else r1
    return turns


def launch_verified(job, tol, max_rounds: int = 12, while_running=None):
    """Launch + boundary check + repair rounds on the observations the job already holds (device work only; see
    ``solve_verified``).  Returns (chunk ids still over tolerance, report); report['kernel_ms'] lists the device time of
    every launch (CUDA events on the job's stream).  ``while_running``: host work to do behind the (asynchronous) first
    launch, before the first wait on the device."""
    job.launch()
    if while_running is not None:
        while_running()
    report = {'rounds': 0, 'repaired_chunks': [], 'boundary_delta_first': None, 'boundary_delta_max': None, 'unverified_chunks': 0,
              'root_branch_chunks': 0}
    kernel_ms = []
    bad = np.zeros(0, dtype=np.int64)
    if job.schedule.chunk_len <= 0 or tol is None:
        job.sync()
        report['kernel_ms'] = [job.kernel_ms()]
        return bad, report
    tol = np.asarray(tol, dtype=np.float64)
    for rnd in range(max_rounds + 1):
        d = job.boundary_deltas()                # on the device, behind the launch; 16 bytes per chunk come back
        kernel_ms.append(job.kernel_ms())
        bad = np.nonzero((d > tol[None]).any(1))[0]
        if rnd == 0:
            report['boundary_delta_first'] = d.max(0).tolist()
            report['chunks_over_tol_first'] = int(len(bad))
        report['boundary_delta_max'] = d.max(0).tolist()
        if not len(bad) or rnd == max_rounds:
            break
        if rnd == 0 and d[:, 0].max() > ROOT_BRANCH_DELTA:
            # chunks on another root branch (root_branch_turns) start again from a cold start on the branch of the
            # sequential pass, all in this one round; the repair rounds below take over from there
            res = job.download()
            turns = root_branch_turns(res.pose[:, :3], (res.status & _lib.ST_SOLVED) != 0, job.chunk_ranges(), job.seq_offsets[:-1])
            ids = np.flatnonzero(turns)
            if len(ids):
                job.relaunch_chunks(ids, job.schedule.chunk_warmup, job.schedule.warmup_full, root_turns=turns[ids])
                report['rounds'] += 1
                report['repaired_chunks'].append(len(ids))
                report['root_branch_chunks'] = int(len(ids))
                continue
        # of a run of consecutive failing chunks only every other one per round, starting with the first
        take, last = [], -2
        for c in bad:
            if c - 1 != last:
                take.append(int(c))
                last = int(c)
        job.relaunch_chunks(take, -1, merge_tol=float(tol[0]) / 3.0)     # merged = a third of the boundary tolerance
        report['rounds'] += 1
        report['repaired_chunks'].append(len(take))
    report['kernel_ms'] = kernel_ms
    return bad, report


def solve_verified(job, obs, vis, *, tol, max_rounds: int = 12, while_running=None):
    """Upload + launch + download, then the boundary check of the chunked schedule and its repair.

    Every chunk reports the state it reached on its last warm-up frame; the emitted result of that frame comes from the
    previous chunk, which is further along its own history.  Where the two differ by more than ``tol`` (root+body pose,
    other pose coefficients, translation, dmpl / expression coefficients) the chunk is solved again in RESUME mode: it
    continues the recursion from the rows the previous chunk emitted, exactly as that chunk would have gone on
    (mosh2_job_relaunch_chunks, chunk_warmup < 0).  A repair round costs one chunk length, not a warm-up.  Neighbouring
    failing chunks are repaired in consecutive rounds (a chunk must not read rows that are being rewritten).  Chunks that
    still fail after ``max_rounds`` keep MOSH2_ST_SHORT_WARMUP on their frames.  Returns (ResultArrays, report)."""
    if obs is not None:          # (None: the caller has uploaded already, e.g. through Job.upload_markers)
        job.upload(obs, vis)
    bad, report = launch_verified(job, tol, max_rounds, while_running)
    res = download_verified(job, bad, report)
    return res, report


def download_verified(job, bad, report):
    """The job's result arrays after ``launch_verified``; the solved frames of the chunks in ``bad`` (still over
    tolerance) carry MOSH2_ST_SHORT_WARMUP."""
    res = job.download()
    if len(bad):
        report['unverified_chunks'] = int(len(bad))
        ranges = job.chunk_ranges()
        for c in bad:
            sl = slice(int(ranges[c, 0]), int(ranges[c, 1]))
            res.status[sl] |= np.where((res.status[sl] & _lib.ST_SOLVED) != 0, _lib.ST_SHORT_WARMUP, 0).astype(res.status.dtype)
        logger.warning('%d chunks did not pass the boundary check after %d repair rounds (max delta %s); their frames carry '
                       'MOSH2_ST_SHORT_WARMUP', len(bad), report['rounds'], report['boundary_delta_max'])
    return res


def _check_mode(mode: str):
    if mode not in BOUNDARY_TOL:
        raise ValueError(f"mode must be 'fast' or 'exact', not {mode!r}")


def _read_capture(fname: str, cfg, latent_labels, labels_map, device_adapter: bool) -> dict:
    """One capture of a Stage-II call: its MocapSession, the selected frames ``sel``, the file column of every latent marker
    ``raw_cols`` (None: host adapter), the host adapter's ``obs`` / ``vis`` and the number of frames ``F``.

    Input adapter.  Normally on the device: the raw marker table of the file goes up as it is and one kernel produces the
    observations and the visibility mask (mosh2_job_upload_markers_range); the host copy of the same clean-up -- needed for
    the output dictionary only -- is made behind the solve.  Labels that own several columns, and frame selections that are
    not a forward range inside the file, take the host path (``frames_for_labels``, obs / vis read here) in front of
    the solve."""
    mocap = MocapSession(fname, mocap_unit=cfg.mocap.unit, mocap_rotate=cfg.mocap.rotate, labels_map=labels_map,
                         only_subjects=[cfg.mocap.subject_name] if cfg.mocap.multi_subject else None)
    labels = list(latent_labels)
    end = len(mocap) if cfg.mocap.end_fidx == -1 else cfg.mocap.end_fidx
    sel = range(cfg.mocap.start_fidx, end, cfg.mocap.ds_rate)                                      # chmosh.py:539-540
    raw_cols = mocap.raw_columns_for_labels(labels) if device_adapter else None
    if raw_cols is not None and not (len(sel) and sel.step > 0 and sel.start >= 0 and sel[-1] < len(mocap)):
        raw_cols = None
    if raw_cols is None:
        obs, vis = mocap.frames_for_labels(labels, sel)
        F = obs.shape[0]
    else:
        obs = vis = None
        F = len(sel)
    if F == 0:
        raise ValueError('no frames selected')
    return dict(fname=fname, cfg=cfg, labels=labels, mocap=mocap, sel=sel, raw_cols=raw_cols, obs=obs, vis=vis, F=F)


def _subject(seqs, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device: int,
             subject_cache: bool = True) -> dict:
    """A subject of a launch: its captures ``seqs`` (``_read_capture``) with its pack, options, flags and device model from
    the subject cache, or with ``subject_cache=False`` prepared for this call alone (``model`` None: ``_solve_launch`` makes
    it and closes it at the end)."""
    if subject_cache:
        pk, opts, flags, model, cache_hit = subject_for(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device)
    else:
        pk, opts, flags = prepare_stageii(cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname)
        model, cache_hit = None, False
    return dict(seqs=seqs, pk=pk, opts=opts, flags=flags, model=model, cache_hit=cache_hit, device=device)


def _resolve_schedule(pk, mode: str, counts, chunk_len, chunk_warmup, warmup_full, first_extra, precision, verify: bool,
                      boundary_tol, sm_budget: int) -> dict:
    """The schedule of one launch over sequences of ``counts`` frames: the keyword overrides of the public entry points over
    the defaults of the pack and ``mode`` (``default_schedule``).  Returns chunk_len (0: one chunk per sequence),
    chunk_warmup, warmup_full, first_extra, precision ('f32' | 'f64'), mode, prec (the MOSH2_* code of the precision) and tol
    (the boundary tolerance; None: no boundary check)."""
    w_def, wf_def, prec_def, tol_def = default_schedule(pk.model_type, mode, pk.n_dmpl)
    chunk_warmup = w_def if chunk_warmup is None else int(chunk_warmup)
    warmup_full = (wf_def if chunk_warmup == w_def else -1) if warmup_full is None else int(warmup_full)
    if first_extra is None:
        first_extra = first_chunk_extra(chunk_warmup, warmup_full)
    if chunk_len is None:
        chunk_len = plan_chunk_len(counts, sm_budget, chunk_warmup, warmup_full if warmup_full >= 0 else chunk_warmup,
                                   first_extra=first_extra)
    if chunk_len >= max(counts):
        chunk_len = 0
    precision = precision or prec_def
    if boundary_tol is None:
        boundary_tol = tol_def
    return dict(chunk_len=chunk_len, chunk_warmup=chunk_warmup, warmup_full=warmup_full, first_extra=first_extra, precision=precision,
                mode=mode, prec={'f32': _lib.MOSH2_F32, 'f64': _lib.MOSH2_F64}[precision], tol=boundary_tol if verify else None)


class _Laps:
    """Host time between consecutive calls, by name (``b200['host_ms']`` of ``mosh_stageii``)."""

    def __init__(self):
        self.ms = {}
        self.t = time.perf_counter()

    def __call__(self, name: str):
        now = time.perf_counter()
        self.ms[name] = self.ms.get(name, 0.0) + (now - self.t) * 1e3
        self.t = now


class _SeqResult:
    """Rows [a, b) of a batch job's ResultArrays: the result arrays of one capture."""

    def __init__(self, res: '_lib.ResultArrays', a: int, b: int):
        for k in ('fullpose', 'pose', 'trans', 'dmpls', 'markers_sim', 'errs', 'status', 'counters'):
            setattr(self, k, getattr(res, k)[a:b].copy())
        self.nd = res.nd


def _solve_launch(subs, sched: dict, t0: float, laps: Optional[_Laps] = None):
    """One verified launch of the captures of the subjects ``subs`` (``_subject``), back to back on the job's frame axis in
    the order given: a batch job of the subject's model (mosh2_job_create_batch) for one subject, a multi-model job
    (mosh2_job_create_multi) for several.  ``sched``: ``_resolve_schedule``.  Every capture uploads its own raw marker table
    into its range of the job (mosh2_job_upload_markers_range); the host-adapter captures go up in one ``job.upload``.

    Returns the per-capture dictionaries, in frame-axis order, each with the capture's own ``b200`` entries (status, counters,
    frame ids, adapter), and the figures of the launch (device time, chunks, schedule, boundary check, totals).  Sets the
    ``offset`` of every capture record on the frame axis.  ``laps``: the host-time laps of ``mosh_stageii``."""
    laps = laps or _Laps()
    seqs = [(sub, s) for sub in subs for s in sub['seqs']]
    counts = [s['F'] for _, s in seqs]
    kw = dict(chunk_len=sched['chunk_len'], chunk_warmup=sched['chunk_warmup'], warmup_full=sched['warmup_full'],
              first_extra=sched['first_extra'], precision=sched['prec'])
    own = [sub for sub in subs if sub['model'] is None]
    for sub in own:
        sub['model'] = _lib.Model(sub['pk'], device=sub['device'])
    laps('model_create_ms')
    try:
        if len(subs) == 1:
            job = subs[0]['model'].job(counts, subs[0]['opts'], **kw)
        else:
            job = _lib.multi_job([sub['model'] for sub in subs], [k for k, sub in enumerate(subs) for _ in sub['seqs']], counts,
                                 subs[0]['opts'], **kw)
        laps('job_create_ms')
        try:
            offsets = job.seq_offsets
            host = [q for q, (_, s) in enumerate(seqs) if s['raw_cols'] is None]
            if len(seqs) == 1 and host:             # one host-adapter capture fills the frame axis
                job.upload(seqs[0][1]['obs'], seqs[0][1]['vis'])
            elif host:
                # host-adapter captures: one upload of the whole frame axis; the device-adapter ranges are written over it
                obs = np.zeros((job.n_frames, subs[0]['pk'].n_markers, 3))
                vis = np.zeros((job.n_frames, subs[0]['pk'].n_markers), dtype=bool)
                for q in host:
                    obs[offsets[q]:offsets[q + 1]], vis[offsets[q]:offsets[q + 1]] = seqs[q][1]['obs'], seqs[q][1]['vis']
                job.upload(obs, vis)
            for q, (_, s) in enumerate(seqs):       # issued back to back: every call stages its own rows
                if s['raw_cols'] is not None:
                    m, rot = s['mocap'], s['cfg'].mocap.rotate
                    job.upload_markers_range(int(offsets[q]), s['F'], m.raw, s['raw_cols'], s['sel'].start, s['sel'].step,
                                             m.unit_per_metre, None if rot is None else _rotation_xyz(rot))
            side = {'ms': 0.0}

            def host_side():                        # the result-independent half of every output, behind the solve
                t_side = time.perf_counter()
                for _, s in seqs:
                    if s['raw_cols'] is not None:
                        s['obs'], s['vis'] = s['mocap'].frames_for_labels(s['labels'], s['sel'])
                    s['lists'] = observation_lists(s['obs'], s['vis'], s['labels'])
                    s['markers_orig'] = s['mocap'].markers[s['sel']]
                side['ms'] = (time.perf_counter() - t_side) * 1e3

            bad, report = launch_verified(job, sched['tol'], while_running=host_side)
            res = download_verified(job, bad, report)
            laps('solve_ms')
            laps.ms['overlapped_host_ms'] = side['ms']
            n_chunks, totals = job.num_chunks, job.totals()
        finally:
            job.close()
    finally:
        for sub in own:
            sub['model'].close()
    laps('close_ms')

    outs = []
    for q, (sub, s) in enumerate(seqs):
        s['offset'] = int(offsets[q])
        r = res if len(seqs) == 1 else _SeqResult(res, int(offsets[q]), int(offsets[q + 1]))
        data = assemble_stageii_data(r, s['obs'], s['vis'], s['labels'], sub['pk'], sub['flags'], bool(sub['opts'].optimize_dynamics),
                                     s['lists'])
        m = s['mocap']
        solved = (r.status & _lib.ST_SOLVED) != 0
        data['stageii_debug_details'].update({
            'markers_orig': s['markers_orig'],
            'labels_orig': m.labels,
            'mocap_fname': s['fname'],
            'mocap_frame_rate': m.frame_rate,
            'mocap_time_length': m.time_length(),
            'b200': {'device_adapter': s['raw_cols'] is not None, 'status': r.status.copy(), 'counters': r.counters.copy(),
                     'pose_reduced': r.pose[solved], 'frame_ids': np.nonzero(solved)[0]},
        })
        outs.append(data)
    laps('assemble_ms')
    n_fb = int(((res.status & _lib.ST_GN_FALLBACK) != 0).sum())
    if n_fb:
        logger.warning('%d frames hit a non-positive-definite Gauss-Newton system (Cauchy step used)', n_fb)
    figures = {'kernel_ms': float(sum(report['kernel_ms'])), 'wall_s': time.time() - t0, 'chunks': n_chunks}
    figures.update({k: sched[k] for k in ('chunk_len', 'chunk_warmup', 'warmup_full', 'first_extra', 'precision', 'mode')})
    figures.update(boundary_check=report, totals=totals)
    return outs, figures


def mosh_stageii(mocap_fname: str, cfg, markers_latent: np.ndarray, latent_labels: list, betas: np.ndarray,
                 marker_meta: dict, v_template_fname=None, *, device: int = 0, mode: str = 'fast',
                 chunk_len: Optional[int] = None, chunk_warmup: Optional[int] = None, warmup_full: Optional[int] = None,
                 first_extra: Optional[int] = None, precision: Optional[str] = None, verify: bool = True, boundary_tol=None,
                 sm_budget: int = NUM_SMS, labels_map='general', subject_cache: bool = True,
                 device_adapter: bool = True) -> dict:
    """Stage II of MoSh++ on one H100.  Positional arguments as in the reference (chmosh.py:458-459).

    Keyword-only extras.  ``mode``: 'fast' (default) = float32, chunked in time with a verified warm-up -- within
    BASELINE.md section 4's tolerances of the reference's sequential float64 result except on the few frames where that
    result is itself ill-conditioned (DESIGN.md section 5); 'exact' = the parity mode: float64, long fully solved
    warm-up, tight boundary check.  ``chunk_len`` (None = planned, 0 = the reference's single sequential pass in one
    thread block), ``chunk_warmup`` / ``warmup_full`` / ``first_extra`` (mosh2_schedule, include/mosh2.h; first_extra None =
    the cost of a warm-up, so that the first chunk finishes with the others), ``precision`` 'f32' | 'f64',
    ``verify`` / ``boundary_tol`` override the mode's presets.  ``labels_map``: 'general' (default) = the synonym table
    the reference always applies (chmosh.py:466), a dict, or None for raw labels.  ``subject_cache``: keep the packed
    per-subject constants and their device copy for the next sequences of the same subject (keyed by the content of every
    input; nothing sequence-dependent is cached).  ``device_adapter``: the mocap input adapter (missing-sample rule, label
    order, units) runs on the GPU from the raw marker table of the file; False = on the host in front of the solve.
    """
    t0 = time.time()
    laps = _Laps()
    _check_mode(mode)
    cap = _read_capture(mocap_fname, cfg, latent_labels, labels_map, device_adapter)
    laps('read_mocap_ms')
    sub = _subject([cap], cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device, subject_cache)
    laps('prepare_ms')
    sched = _resolve_schedule(sub['pk'], mode, [cap['F']], chunk_len, chunk_warmup, warmup_full, first_extra, precision, verify,
                              boundary_tol, sm_budget)
    laps('dense_view_ms')
    (data,), figures = _solve_launch([sub], sched, t0, laps)
    if cap['raw_cols'] is not None:             # the table rows the selection spans (float64) and the column map
        h2d = ((cap['F'] - 1) * cap['sel'].step + 1) * cap['mocap'].raw.shape[1] * 24 + 4 * len(cap['labels'])
    else:
        h2d = cap['obs'].size * (4 if sched['precision'] == 'f32' else 8) + cap['vis'].size
    data['stageii_debug_details']['b200'].update(figures, host_ms=laps.ms, subject_cache_hit=sub['cache_hit'], h2d_bytes=int(h2d))
    return data


def mosh_stageii_batch(mocap_fnames, cfg, markers_latent: np.ndarray, latent_labels: list, betas: np.ndarray, marker_meta: dict,
                       v_template_fname=None, *, device: int = 0, mode: str = 'fast', chunk_len: Optional[int] = None,
                       chunk_warmup: Optional[int] = None, warmup_full: Optional[int] = None, first_extra: Optional[int] = None,
                       precision: Optional[str] = None, verify: bool = True, boundary_tol=None, sm_budget: int = NUM_SMS,
                       labels_map='general', subject_cache: bool = True, device_adapter: bool = True) -> list:
    """Stage II of several captures of ONE subject (one Stage-I result, one ``cfg`` apart from ``mocap.fname``) in one launch.

    Returns one dictionary per capture, in the order of ``mocap_fnames``: what ``mosh_stageii`` returns for that capture with
    the same keyword arguments, except ``stageii_debug_details['b200']``.  The captures share one pack (subject cache) and one
    batch job (mosh2_job_create_batch): their frames lie back to back on the job's frame axis, the chunk length is planned
    over all their frame counts (``plan_chunk_len``, as ``shard.GpuRankSolver`` does), and one verified launch with its
    repair rounds (``launch_verified``) and one download serve them all.  Every capture uploads its own raw marker table
    into its range of the job (mosh2_job_upload_markers_range); a capture whose labels own several columns or whose frame
    selection is not a forward range takes the host adapter, as in ``mosh_stageii``.  ``b200`` holds the capture's own
    status / counters / frame ids and, under ``'batch'``, the figures of the whole launch (device time, chunks, boundary
    check, totals), marked ``'shared': True`` -- the same for every capture of the call."""
    t0 = time.time()
    _check_mode(mode)
    seqs = [_read_capture(fn, cfg, latent_labels, labels_map, device_adapter) for fn in mocap_fnames]
    if not seqs:
        raise ValueError('no captures given')
    sub = _subject(seqs, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname, device, subject_cache)
    counts = [s['F'] for s in seqs]
    sched = _resolve_schedule(sub['pk'], mode, counts, chunk_len, chunk_warmup, warmup_full, first_extra, precision, verify,
                              boundary_tol, sm_budget)
    outs, figures = _solve_launch([sub], sched, t0)
    batch = {'shared': True, 'captures': len(seqs), 'frames': int(sum(counts)), **figures, 'subject_cache_hit': sub['cache_hit']}
    for q, (s, data) in enumerate(zip(seqs, outs)):
        data['stageii_debug_details']['b200'].update(batch=batch, batch_index=q, frame_offset=s['offset'])
    return outs


def kernel_shape_key(pk) -> tuple:
    """What two packs must share to be solved by one multi-model launch (mosh2_job_create_multi): sizes, free-variable
    counts, finger / face / joint-angle ranges, prior size and the hand-block structure of the hand-PCA matrix (the non-zero
    column range of every row).  The tables themselves may differ."""
    hc = np.asarray(pk.hand_comps).reshape(pk.n_hand_red, pk.n_hand_full) if pk.n_hand_red else np.zeros((0, 0))
    rows = []
    for r in hc:
        nz = np.flatnonzero(r)
        rows.append((int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0))
    return (pk.n_joints, pk.n_markers, pk.body_dof, pk.p_red, pk.n_hand_red, pk.n_hand_full, pk.n_dmpl, pk.kw, len(pk.free_step1),
            len(pk.free_step2), pk.finger_lo, pk.finger_hi, pk.n_expr, pk.face_lo, pk.face_hi, len(getattr(pk, 'jangles_ids', ())),
            pk.prior_k, pk.prior_d, tuple(rows))


def subject_launch_key(pk, opts, mode: str = 'fast') -> tuple:
    """Subjects with equal keys share a launch of ``mosh_stageii_subjects``: one kernel shape (``kernel_shape_key``), equal
    ``mosh2_options`` and the same default schedule (``default_schedule``: precision, warm-up, boundary tolerance)."""
    return (kernel_shape_key(pk), tuple(getattr(opts, f) for f, _ in opts._fields_), default_schedule(pk.model_type, mode, pk.n_dmpl))


def launch_groups(keys) -> list:
    """Subjects (by their ``subject_launch_key``) that share a launch: lists of subject indices, in the order of first
    appearance."""
    groups = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    return list(groups.values())


def mosh_stageii_subjects(subjects, *, device: int = 0, mode: str = 'fast', chunk_len: Optional[int] = None,
                          chunk_warmup: Optional[int] = None, warmup_full: Optional[int] = None, first_extra: Optional[int] = None,
                          precision: Optional[str] = None, verify: bool = True, boundary_tol=None, sm_budget: int = NUM_SMS,
                          labels_map='general', device_adapter: bool = True) -> list:
    """Stage II of the captures of SEVERAL subjects, with as few launches as their models allow.

    ``subjects``: dictionaries with ``cfg``, ``mocap_fnames`` and the subject's Stage-I outputs ``markers_latent``,
    ``latent_labels``, ``betas``, ``marker_meta`` and (optional) ``v_template_fname``.  Returns one list per subject with one
    dictionary per capture: what ``mosh_stageii_batch`` returns for that subject with the same keyword arguments, except
    ``stageii_debug_details['b200']`` and, in the planned (``chunk_len=None``) schedule, the chunk length, which is planned over
    all frame counts of the launch.

    Every subject's pack and device model come from the subject cache (``subject_for``).  Subjects whose packs have one kernel
    shape (``kernel_shape_key``) and whose ``mosh2_options`` and default schedule (``default_schedule``: precision, warm-up,
    boundary tolerance) are equal share one multi-model job (mosh2_job_create_multi) and one verified launch
    (``launch_verified``); e.g. male and female SMPL-H subjects share a launch, a DMPL subject (float64 exact preset) does not
    share one with float32 SMPL-H subjects.  ``b200['batch']`` holds the figures of the capture's launch, marked
    ``'shared': True``, and ``'launches'``, the number of launches of the call."""
    global SUBJECT_CACHE_SIZE
    t0 = time.time()
    _check_mode(mode)
    subjects = list(subjects)
    bound = SUBJECT_CACHE_SIZE
    SUBJECT_CACHE_SIZE = max(bound, len(subjects))      # (every model of the call stays open until its launch is done)
    try:
        subs = []
        for s in subjects:
            seqs = [_read_capture(fn, s['cfg'], s['latent_labels'], labels_map, device_adapter) for fn in s['mocap_fnames']]
            if not seqs:
                raise ValueError('a subject without captures')
            subs.append(_subject(seqs, s['cfg'], s['markers_latent'], s['latent_labels'], s['betas'], s['marker_meta'],
                                 s.get('v_template_fname'), device))
        groups = launch_groups([subject_launch_key(sub['pk'], sub['opts'], mode) for sub in subs])
        out = [[] for _ in subs]
        for g, members in enumerate(groups):
            group = [subs[i] for i in members]
            counts = [s['F'] for sub in group for s in sub['seqs']]
            sched = _resolve_schedule(group[0]['pk'], mode, counts, chunk_len, chunk_warmup, warmup_full, first_extra, precision,
                                      verify, boundary_tol, sm_budget)
            outs, figures = _solve_launch(group, sched, t0)
            batch = {'shared': True, 'launch': g, 'launches': len(groups), 'subjects': len(group), 'captures': len(counts),
                     'frames': int(sum(counts)), **figures, 'subject_cache_hits': [sub['cache_hit'] for sub in group]}
            seqs = [(k, i, s) for k, i in enumerate(members) for s in subs[i]['seqs']]
            for q, ((k, i, s), data) in enumerate(zip(seqs, outs)):
                data['stageii_debug_details']['b200'].update(batch=batch, batch_index=q, subject_index=k, frame_offset=s['offset'])
                out[i].append(data)
    finally:
        SUBJECT_CACHE_SIZE = bound
        while len(_SUBJECT_CACHE) > SUBJECT_CACHE_SIZE:
            _, old = _SUBJECT_CACHE.popitem(last=False)
            old['model'].close()
    return out
