"""``mosh_stagei`` -- Stage I of MoSh++ (shape, latent markers, the poses of the picked frames) on libmosh2.so (H100).

Reference: src/moshpp/chmosh.py:83-455 (SURVEY.md 8(f-2)).  Same inputs (``stagei_frames``: one ``{label: xyz}`` dictionary
per picked frame, ``cfg``, ``betas_fname``, ``v_template_fname``) and the same return dictionary (chmosh.py:436-455).  The
marker layout comes from ``cfg.dirs.marker_layout.fname`` (``load_marker_layout`` reads the reference's json, chmosh.py:121-125)
or is passed in loaded (``marker_meta``); creating layouts is outside this build (SURVEY.md section 2).

What runs where
  device   per picked frame (one thread block each, ``mosh2_job_linearize``): SMPL forward, simulated markers, the residuals of
           the frame's own terms (data, pose prior, fingers), their normal equations and the Jacobian rows of the data term --
           wrt the frame's pose / translation AND wrt the shape coefficients (the shape directions ride as the linear block of
           the Stage-II kernel); the closest-point search and the point-to-triangle distances + derivatives of the surface
           term (``mosh2_mesh_distance``);
  host     the chumpy graph around them that couples the frames: marker attachment on the canonical body (8-NN local frames,
           re-made whenever the latent markers or the shape move, transformed_lm.py:59-113), the chain through the attachment
           coefficients, the init / shape-prior / surface terms' small Jacobians, the block-arrow normal equations
           (12 x ~100 private unknowns + 3 M + num_betas shared ones) and chumpy's dog-leg on them, float64.
There is no CPU evaluation of the body model per frame: without libmosh2.so or a GPU the call raises.

The canonical body ``can_model.r`` (zero reduced pose: with ``use_hands_mean`` the hands are in their mean pose) is an affine
function of the shape coefficients -- rotations fixed, joints and vertices linear in betas -- so it is expanded once:
can(betas) = can_0 + C betas[:num_betas] (``CanonicalBody``).

``moshpp.optimize_face`` (SMPL-X with face markers, the shape given and ``optimize_betas`` off; chmosh.py:103-151,283-295):
every picked frame's model carries the given shape plus its own expressions ``betas[es:es + ne]``; the canonical body keeps
zero expressions.  The device's linear block then holds the expression directions instead of the shape's, and in the two
detailed steps the jaw and the expressions are private unknowns of each frame, with the poseF / expr terms.  The expressions
are returned in the debug details as ``opt_models_expression``.

``face_with_free_shape`` (SMPL-X with face markers, ``optimize_betas`` and ``optimize_face``; the reference raises here): the
union of the two objectives.  Each frame's model carries the free shape plus its own expressions, the canonical body the shape
with zero expressions; the linear block holds the shape directions followed by the expression directions.  The shape columns
stay shared (attachment, init, surface and beta terms as with a free shape), the expressions private to their frame.

``reference_options`` (off by default: either option raises): the head-marker correlation prior replaces the init terms of
the correlated markers by ``corr (ml - init)[head_ids]``, dense over their latent unknowns in the shared block; the extra
initial rigid adjustment is one dog-leg over every frame's root orientation and translation on the unweighted data term, its
normal equations 6 x 6 blocks from the same device linearisation with no shared block (DESIGN.md section 10).

``robust_data_sigma`` (None by default: least squares): every data row of the four annealing steps and of the extra rigid
adjustment becomes wd psi(e), the Geman-McClure row of Stage II (psi(e) = sigma e / sqrt(sigma^2 + e^2) per coordinate of a
visible marker's e = sim - obs).  The device returns those rows and its own Jacobian columns robust already; the host scales the
columns it adds through the attachment (latent markers, the shape's attachment part) by the same psi', recovered from the
stored rows as the kernel does (``data_dpsi_gm``).  The Procrustes start and every other term stay least squares.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Optional

import numpy as np

from . import lib as _lib
from . import mesh_distance as _md
from . import pack as _pack
from .chmosh import _get, _read_vertices, check_robust_sigma

logger = logging.getLogger('moshpp_b200')
NUM_TRAIN_MARKERS = 46      # chmosh.py:100


# ---------------------------------------------------------------------------------------------------------------------
# marker layout file (the json the reference's Stage I reads, marker_layout/edit_tools.py:83-183)
# ---------------------------------------------------------------------------------------------------------------------
def load_marker_layout(marker_layout_fname: str, labels_map='general', exclude_marker_types=None, exclude_markers=None,
                       only_markers=None) -> dict:
    """``marker_layout_load`` (marker_layout/edit_tools.py:83-183): marker types sorted by name, labels sorted within a type
    (after the synonym map), ``marker_vids`` / ``marker_type`` / ``marker_type_mask`` / ``m2b_distance`` /
    ``surface_model_type``.  As in the reference, ``exclude_markers`` is only logged there (:150-151, no ``continue``) and has
    no effect; colours are a plain red-to-blue ramp (the reference uses the ``colour`` package; viewers only)."""
    import json
    from collections import OrderedDict
    from .mocap_interface import general_labels_map
    assert str(marker_layout_fname).endswith('.json')
    with open(marker_layout_fname) as f:
        d = json.load(f)
    if isinstance(labels_map, str):
        labels_map = general_labels_map()
    only_markers = only_markers or []
    exclude_marker_types = exclude_marker_types or []
    marker_vids, marker_types, m2b = OrderedDict(), OrderedDict(), OrderedDict()
    for ms in sorted(d['markersets'], key=lambda a: a['type']):
        t = ms['type']
        if t in exclude_marker_types:
            continue
        if t in m2b:
            raise ValueError(f'Marker type appears in multiple occasions: {t}!')
        m2b[t] = ms.get('distance_from_skin', 0.0095)
        cur = ms['indices']
        if labels_map:
            cur = {labels_map.get(k, k): cur[k] for k in cur}
        for label in sorted(cur):
            if only_markers and label not in only_markers:
                continue
            if label in marker_vids:
                raise ValueError(f'Label ({label}) is present in multiple occasions.')
            marker_vids[label] = int(cur[label])
            marker_types.setdefault(t, []).append(label)
    mask = OrderedDict((k, np.array([l in marker_types[k] for l in marker_vids.keys()])) for k in marker_types)
    mtype = OrderedDict()
    for i, l in enumerate(marker_vids):
        for k, m in mask.items():
            if m[i]:
                mtype[l] = k
    n = max(1, len(marker_vids) - 1)
    colors = OrderedDict((l, [1.0 - i / n, 0.0, i / n]) for i, l in enumerate(marker_vids))
    colors['nan'] = [0.83, 1, 0]
    return {'marker_vids': marker_vids, 'marker_colors': colors, 'marker_type': mtype, 'marker_type_mask': mask, 'm2b_distance': m2b,
            'surface_model_type': d.get('surface_model_type', 'smplx'), 'marker_layout_fname': marker_layout_fname}


def write_marker_layout(fname: str, marker_meta: dict) -> str:
    """The marker layout json the reference's Stage I reads (marker_layout/edit_tools.py:115-160) from a ``marker_meta``
    (``marker_layout_write`` without the colours and the viewer files)."""
    import json
    sets = []
    for t, mask in marker_meta['marker_type_mask'].items():
        labels = [l for l, m in zip(marker_meta['marker_vids'].keys(), np.asarray(mask, dtype=bool)) if m]
        sets.append({'type': t, 'distance_from_skin': float(marker_meta['m2b_distance'][t]),
                     'indices': {l: int(marker_meta['marker_vids'][l]) for l in labels}})
    with open(fname, 'w') as f:
        json.dump({'surface_model_type': marker_meta['surface_model_type'], 'markersets': sets}, f)
    return fname


# ---------------------------------------------------------------------------------------------------------------------
# small host-side geometry (float64 numpy, O(markers))
# ---------------------------------------------------------------------------------------------------------------------
def _skew(v):
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def _dnrm(u):
    """d (u / |u|) / du for rows of u: (I - uh uh^T) / |u|."""
    n = np.linalg.norm(u, axis=1)
    uh = u / n[:, None]
    return (np.eye(3)[None] - uh[:, :, None] * uh[:, None, :]) / n[:, None, None]


def local_frames(v0, v1, v2):
    """Rows f1, f2, f3 of the marker frames on the triples (transformed_lm.py:84-101,139-150) and their derivatives wrt the
    edge vectors e1 = v1 - v0, e2 = v2 - v0: F [M,3,3] (rows), dF/de1, dF/de2 [M,3(row),3,3]."""
    e1, e2 = v1 - v0, v2 - v0
    n = np.cross(e1, e2)
    f1 = e1 / np.linalg.norm(e1, axis=1, keepdims=True)
    f2 = n / np.linalg.norm(n, axis=1, keepdims=True)
    f3 = np.cross(f1, f2)
    df1_de1 = _dnrm(e1)
    df2_de1 = -np.einsum('mij,mjk->mik', _dnrm(n), _skew(e2))
    df2_de2 = np.einsum('mij,mjk->mik', _dnrm(n), _skew(e1))
    df3_de1 = -np.einsum('mij,mjk->mik', _skew(f2), df1_de1) + np.einsum('mij,mjk->mik', _skew(f1), df2_de1)
    df3_de2 = np.einsum('mij,mjk->mik', _skew(f1), df2_de2)
    F = np.stack([f1, f2, f3], 1)
    dF1 = np.stack([df1_de1, df2_de1, df3_de1], 1)
    dF2 = np.stack([np.zeros_like(df1_de1), df2_de2, df3_de2], 1)
    return F, dF1, dF2


def attachment_coefficients(tri_verts, ml):
    """k = F (ml - v0) on the canonical triples [M,3,3] and d k / d (v0, v1, v2) [M,3,9] (d k / d ml = F)."""
    v0, v1, v2 = tri_verts[:, 0], tri_verts[:, 1], tri_verts[:, 2]
    F, dF1, dF2 = local_frames(v0, v1, v2)
    d = ml - v0
    k = np.einsum('mij,mj->mi', F, d)
    dk_de1 = np.einsum('mj,mijk->mik', d, dF1)
    dk_de2 = np.einsum('mj,mijk->mik', d, dF2)
    dk_dv = np.concatenate([-F - dk_de1 - dk_de2, dk_de1, dk_de2], axis=2)
    return k, F, dk_dv


def marker_points(tri_verts, k):
    """v0 + F^T k (transformed_lm.py:155-158) and its derivative wrt (v0, v1, v2) [M,3,9]."""
    v0, v1, v2 = tri_verts[:, 0], tri_verts[:, 1], tri_verts[:, 2]
    F, dF1, dF2 = local_frames(v0, v1, v2)
    pts = v0 + np.einsum('mij,mi->mj', F, k)
    d_e1 = np.einsum('mi,mijk->mjk', k, dF1)
    d_e2 = np.einsum('mi,mijk->mjk', k, dF2)
    eye = np.broadcast_to(np.eye(3), d_e1.shape)
    return pts, np.concatenate([eye - d_e1 - d_e2, d_e1, d_e2], axis=2)


def vertex_normals(v, f):
    """Normalised sum of the area-scaled triangle normals around every vertex (scan2mesh/ch_vert_normals.py:86-139)."""
    tn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    vn = np.stack([np.bincount(f.reshape(-1), weights=np.repeat(tn[:, c], 3), minlength=len(v)) for c in range(3)], axis=1)
    ss = (vn ** 2).sum(1)
    ss[ss == 0] = 1e-10
    return vn / np.sqrt(ss)[:, None]


def rigid_fit(sim, obs):
    """rigid_transformations.py:39-83: R, T = argmin |R sim + T - obs| (SVD, det fix) -> (axis-angle of R, T)."""
    ca, cb = sim.mean(0), obs.mean(0)
    H = (sim - ca).T.dot(obs - cb)
    U, _, Vt = np.linalg.svd(H)
    R = Vt.T.dot(U.T)
    if np.linalg.det(R) < 0:
        Vt[2] *= -1
        R = Vt.T.dot(U.T)
    T = cb - R.dot(ca)
    cos = np.clip((np.trace(R) - 1.0) / 2.0, -1.0, 1.0)
    th = np.arccos(cos)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if th < 1e-8:
        rv = 0.5 * w
    elif np.pi - th < 1e-6:                       # near pi: the axis from the symmetric part
        Bm = (R + np.eye(3)) / 2.0
        ax = np.sqrt(np.maximum(np.diag(Bm), 0.0))
        i = int(np.argmax(ax))
        ax = Bm[i] / ax[i]
        if w.dot(ax) < 0:
            ax = -ax
        rv = th * ax / np.linalg.norm(ax)
    else:
        rv = th / (2.0 * np.sin(th)) * w
    return rv, T


def _solve_arrow(A, g, ns, n_p, F):
    """A d = g for the block-arrow normal equations [[S, B^T], [B, blockdiag(D_f)]]: shared unknowns first (ns), then F
    private blocks of n_p -- by the Schur complement of the private blocks (each picked frame couples to the others only
    through the shape and the latent markers).  Falls back to chumpy's dense solve / lstsq when a block is singular
    (SURVEY.md A.6)."""
    try:
        S = A[:ns, :ns].copy()
        gs = g[:ns].copy()
        X = []
        for f in range(F):
            sl = slice(ns + f * n_p, ns + (f + 1) * n_p)
            B = A[sl, :ns]
            Xf = np.linalg.solve(A[sl, sl], np.concatenate([B, g[sl, None]], axis=1))
            S -= B.T.dot(Xf[:, :ns])
            gs -= B.T.dot(Xf[:, ns])
            X.append(Xf)
        ds = np.linalg.solve(S, gs)
        return np.concatenate([ds] + [Xf[:, ns] - Xf[:, :ns].dot(ds) for Xf in X])
    except np.linalg.LinAlgError:
        try:
            return np.linalg.solve(A, g)
        except np.linalg.LinAlgError:
            return np.linalg.lstsq(A, g, rcond=None)[0]


def data_dpsi_gm(r, wd, sigma):
    """psi'(e) of the Geman-McClure data rows r = wd psi(e), recovered from the rows alone by the kernel's rule
    (csrc/mosh2_device.cuh ``data_dpsi_gm``): u = r / (wd sigma) = e / sqrt(sigma^2 + e^2), psi' = (1 - u^2)^(3/2) clamped at
    0, and 0 where the row is exactly 0 (e = 0, or an invisible marker)."""
    u = r / (wd * sigma)
    t = np.maximum(1.0 - u * u, 0.0)
    return np.where(r != 0, t * np.sqrt(t), 0.0)


class CanonicalBody:
    """can(betas) = can_0 + C betas[:nb]: the canonical mesh as an affine function of the free shape coefficients."""

    def __init__(self, model: _pack.SurfaceModel, betas_all: np.ndarray, nb: int):
        def can(b):
            v_shaped = model.v_template + model.shapedirs[:, :, :len(b)].dot(b)
            return _pack.canonical_verts(model, v_shaped, model.J_regressor.dot(v_shaped))
        b0 = np.array(betas_all, dtype=np.float64)
        b0[:nb] = 0.0
        self.base = can(b0)
        self.C = np.zeros(self.base.shape + (nb,))
        for i in range(nb):
            b = b0.copy()
            b[i] = 1.0
            self.C[:, :, i] = can(b) - self.base

    def __call__(self, betas_free):
        return self.base + self.C.dot(betas_free)


# ---------------------------------------------------------------------------------------------------------------------
# device back end
# ---------------------------------------------------------------------------------------------------------------------
class DeviceBackend:
    """The two device services Stage I uses.  Tests substitute a back end built on the host build of the same device source."""

    def __init__(self, device: int = 0):
        self.device = device
        _lib.load_library()

    def linearize(self, pk, options, obs, vis, x, step, build):
        model = _lib.Model(pk, device=self.device)
        try:
            job = model.job(obs.shape[0], options, chunk_len=1, chunk_warmup=0, precision=_lib.MOSH2_F64)
            try:
                job.upload(obs, vis)
                return job.linearize(x, options, step, build)
            finally:
                job.close()
        finally:
            model.close()

    def squared_distance(self, samples, verts, faces):
        out = _md.mesh_distance(samples, verts, faces, kind='squared', device=self.device)
        return out['value'], out['tri'], out['part'], out['d_sample'], out['d_tri']


# ---------------------------------------------------------------------------------------------------------------------
# the solver
# ---------------------------------------------------------------------------------------------------------------------
def face_flag(cfg, marker_meta, avail_labels, face_with_free_shape: bool = False) -> bool:
    """Whether Stage I fits the jaw and the expressions (``moshpp.optimize_face``), by the reference's rules, without changing
    ``cfg``: off with a free shape when the face markers are excluded (chmosh.py:103-118), off without a face-type marker in the
    layout or without a face label in the picked frames (chmosh.py:127-137), ignored for models other than SMPL-X (only SMPL-X has
    a jaw and expression components), and NotImplementedError with a free shape on SMPL-X (chmosh.py:287-291) unless
    ``face_with_free_shape`` asks for the joint fit of the shape and every picked frame's expressions."""
    sm, mp = cfg.surface_model, cfg.moshpp
    if not bool(_get(mp, 'optimize_face', False)):
        return False
    free_betas = bool(mp.optimize_betas)
    if sm.type == 'smplx' and free_betas and 'face' in (_get(cfg.mocap, 'exclude_marker_types', None) or []):
        return False
    if not np.any(['face' in t for t in marker_meta['marker_type_mask'].keys()]):
        return False
    if not np.any([('face' in t) and l in avail_labels for l, t in marker_meta['marker_type'].items()]):
        return False
    if sm.type != 'smplx':
        return False
    if free_betas and not face_with_free_shape:
        raise NotImplementedError('optimize_face with optimize_betas: Stage I fits per-frame expressions with a free shape only '
                                  'when asked to (face_with_free_shape=True); otherwise give the shape (betas_fname or '
                                  'v_template_fname) with optimize_betas off (chmosh.py:287-291)')
    return True


class StageI:
    def __init__(self, stagei_frames, cfg, marker_meta, betas=None, v_template=None, backend=None, *,
                 face_with_free_shape: bool = False, reference_options: bool = False, robust_data_sigma=None):
        sm, mp = cfg.surface_model, cfg.moshpp
        self.robust_sigma = check_robust_sigma(robust_data_sigma)           # None: the least-squares data term
        self.cfg, self.marker_meta = cfg, marker_meta
        self.backend = backend or DeviceBackend()
        self.labels = list(marker_meta['marker_vids'].keys())
        M = self.M = len(self.labels)
        F = self.F = len(stagei_frames)
        avail = set(k for fr in stagei_frames for k in fr.keys())
        self.fingers = bool(mp.optimize_fingers)
        if self.fingers:                                                                           # chmosh.py:130-141
            if not np.any(['finger' in m for m in marker_meta['marker_type_mask'].keys()]):
                self.fingers = False
            elif not np.any([('finger' in t) and l in avail for l, t in marker_meta['marker_type'].items()]):
                self.fingers = False
        self.free_betas = bool(mp.optimize_betas)
        self.face = face_flag(cfg, marker_meta, avail, face_with_free_shape)
        self.reference_options = reference_options
        # the head-marker correlation prior (chmosh.py:252-266): head_ids / head_corr stay None when it does not apply
        self.head_ids, self.head_corr = None, None
        corr_fname = _get(mp, 'head_marker_corr_fname', None)
        if corr_fname is not None:
            if not reference_options:
                raise NotImplementedError('moshpp.head_marker_corr_fname (chmosh.py:252-266,360-373) applies only when asked to '
                                          '(reference_options=True); otherwise set it to None')
            head_meta = np.load(corr_fname)
            head_labels = [str(l) for l in head_meta['mrk_labels']]
            missing = [l for l in head_labels if l not in marker_meta['marker_vids']]
            if missing:
                logger.debug(f'not all of the head markers are in the layout, the head-marker correlation is not used: {missing}')
            else:
                self.head_ids = [self.labels.index(l) for l in head_labels]
                self.head_corr = np.asarray(head_meta['corr'], dtype=np.float64)                # K x H
        self.model = model = _pack.load_surface_model(sm.fname, pose_hand_prior_fname=_get(mp, 'pose_hand_prior_fname'),
                                                      use_hands_mean=bool(sm.use_hands_mean), dof_per_hand=int(sm.dof_per_hand),
                                                      v_template=v_template, surface_model_type=sm.type)
        if model.faces is None:
            raise ValueError('the body model has no faces: Stage I needs the mesh for its surface term')
        self.faces = np.asarray(model.faces, dtype=np.int64)
        self.prior = None
        pf = _get(mp, 'pose_body_prior_fname')
        if pf and model.model_type == 'animal_horse':
            self.prior = _pack.create_horse_body_prior(pf)
        elif pf and model.model_type == 'animal_dog':
            self.prior = _pack.create_dog_body_prior(pf)
        elif pf and model.model_type != 'mano':
            self.prior = _pack.create_gmm_body_prior(pf, exclude_hands=model.model_type in ('smplh', 'smplx'))
        self.nb = int(sm.num_betas)
        self.betas = np.zeros(model.shapedirs.shape[-1])
        if betas is not None:
            self.betas[:self.nb] = np.asarray(betas)[:self.nb]                                   # chmosh.py:169-172
        self.can = CanonicalBody(model, self.betas, self.nb)
        self.jd_lin = np.einsum('jv,vcd->jcd', model.J_regressor, model.shapedirs[:, :, :self.nb])    # joint directions of the shape block
        self.pose = np.zeros((F, model.p_red))
        self.trans = np.zeros((F, 3))
        # optimize_face: each picked frame's expression coefficients, betas[es:es + ne] of its own model (chmosh.py:136-151,292-294)
        self.es = int(_get(sm, 'betas_expr_start_id', 0) or 0) if self.face else 0
        self.ne = int(_get(sm, 'num_expressions', 0) or 0) if self.face else 0
        self.expr = np.zeros((F, self.ne))

        can_v = self.can(self.betas[:self.nb])                                                   # chmosh.py:57-82
        vn = vertex_normals(can_v, self.faces)
        self.m2b = np.ones(M) * 0.0095
        for t, mask in marker_meta['marker_type_mask'].items():
            self.m2b[np.asarray(mask, dtype=bool)] = marker_meta['m2b_distance'][t]
        vids = np.asarray(list(marker_meta['marker_vids'].values()), dtype=np.int64)
        self.ml = can_v[vids] + vn[vids] * self.m2b[:, None]
        self.closest0, self.k0 = _pack.attach_markers(can_v, self.ml)                            # tc2: constants (chmosh.py:185)

        self.obs = np.zeros((F, M, 3))
        self.vis = np.zeros((F, M), dtype=bool)
        for f, fr in enumerate(stagei_frames):                                                   # chmosh.py:193-206
            for i, l in enumerate(self.labels):
                if l in fr and not np.any(np.isnan(fr[l])):
                    self.obs[f, i], self.vis[f, i] = fr[l], True
        self.stats = dict(evaluations=0, linearisations=0, iterations=0, minimisations=0)

    # ---- device pack of the current (betas, latent markers): the Stage-II constants with the shape directions as linear block
    def pack_for(self, detailed: bool, can_v=None):
        sm, mp = self.cfg.surface_model, self.cfg.moshpp
        toes = bool(_get(mp, 'optimize_toes', False))
        if self.face and not self.free_betas:
            # the shape is given: the linear block is the expression directions alone, and Step 2 frees the jaw and them
            return _pack.build_pack(self.model, self.betas, self.ml, num_betas=self.nb, prior=self.prior,
                                    optimize_fingers=self.fingers, optimize_toes=toes, optimize_face=True,
                                    expr_start=self.es, num_expressions=self.ne, can_verts=can_v)
        # the linear block is the shape directions, followed by the expression directions when the face is fitted with the
        # shape (face_with_free_shape); the free lists keep a frame's own unknowns first and the shared shape columns last
        pk = _pack.build_pack(self.model, self.betas, self.ml, num_betas=self.nb, prior=self.prior,
                              dmpl_dirs=self.model.shapedirs[:, :, :self.nb], num_dmpls=self.nb,
                              optimize_fingers=self.fingers, optimize_toes=toes, optimize_face=self.face,
                              expr_start=self.es, num_expressions=self.ne, can_verts=can_v, jd_lin=self.jd_lin)
        lo = 3 + pk.p_red
        lin = [lo + i for i in range(self.nb)] if self.free_betas else []
        s1 = [int(i) for i in pk.free_step1 if i < lo]
        s2 = [int(i) for i in pk.free_step2 if i < lo or i >= lo + self.nb]       # trans | pose ids | expressions
        pk.free_step1 = np.asarray(s1 + lin, dtype=np.int32)
        pk.free_step2 = np.asarray(s2 + lin, dtype=np.int32)
        return pk

    def weights_for(self, anneal):
        w = self.cfg.opt_settings.weights
        out = {'poseB': w['stagei_wt_poseB'] * anneal, 'poseH': w['stagei_wt_poseH'] * anneal, 'beta': w['stagei_wt_betas'] * anneal,
               'data': (w['stagei_wt_data'] / anneal) * (NUM_TRAIN_MARKERS / self.M), 'surf': w['stagei_wt_surf'], 'init': {}}
        for k in self.marker_meta['marker_type_mask'].keys():
            try:
                base = w[f'stagei_wt_init_{k}']
            except (KeyError, AttributeError):
                base = w['stagei_wt_init']
            out['init'][k] = base * anneal
        if self.head_ids is not None:       # the body type's init weight, else the base one (chmosh.py:368-369)
            out['init_head_corr'] = out['init'].get('body', w['stagei_wt_init'] * anneal)
        if self.face:                                                                               # chmosh.py:322-324
            out['poseF'], out['expr'] = w['stagei_wt_poseF'] * anneal, w['stagei_wt_expr'] * anneal
        return out

    # ---- one evaluation of the whole objective; with want_jac also its block-arrow normal equations ---------------------
    def evaluate(self, want_jac: bool, wts, detailed: bool):
        M, F, nb = self.M, self.F, (self.nb if self.free_betas else 0)
        self.stats['evaluations'] += 1
        self.stats['linearisations'] += int(want_jac)
        can_v = self.can(self.betas[:self.nb])
        pk = self.pack_for(detailed, can_v)
        step = 2 if detailed else 1
        free = pk.free_step2 if detailed else pk.free_step1
        n_f = len(free)
        n_p = n_f - nb
        x = np.zeros((F, pk.nx))
        x[:, :3], x[:, 3:3 + pk.p_red] = self.trans, self.pose
        if self.face:           # (the shape slots of the linear block stay zero: the pack's rest vertices carry the shape)
            x[:, 3 + pk.p_red + pk.n_dmpl - pk.n_expr:] = self.expr
        opts = _lib.make_options(None, optimize_fingers=detailed and self.fingers and pk.finger_hi > pk.finger_lo,
                                 optimize_face=detailed and self.face)
        opts.wt_data, opts.wt_poseB, opts.wt_poseH = float(wts['data']), float(wts['poseB']), float(wts['poseH'])
        if self.face:
            opts.wt_poseF, opts.wt_expr = float(wts['poseF']), float(wts['expr'])
        if self.robust_sigma is not None:
            opts.robust_sigma = self.robust_sigma
        dev = self.backend.linearize(pk, opts, self.obs, self.vis, x, step, want_jac)
        sse = {'data': float(dev['errs'][:, 0].sum())}
        if pk.prior_k:
            sse['poseB'] = float(dev['errs'][:, 1].sum())
            if len(pk.jangles_ids):         # the horse's joint-angle term (chmosh.py:358-360); the kernel reports it in poseH
                sse['poseB_jangles'] = float(dev['errs'][:, 3].sum())
        if detailed and self.fingers:
            sse['poseH'] = float(dev['errs'][:, 3].sum())
        if detailed and self.face:
            sse['poseF'] = float(dev['errs'][:, 6].sum())
            sse['expr'] = float(dev['errs'][:, 7].sum())

        # init: the latent markers against the initial guess riding on the current canonical body (chmosh.py:185-186,362)
        init, dinit_dv = marker_points(can_v[self.closest0], self.k0)
        r_init = self.ml - init
        w_init = np.zeros(M)
        for k, mask in self.marker_meta['marker_type_mask'].items():
            mask = np.asarray(mask, dtype=bool)
            if self.head_ids is not None:
                # with the head-marker correlation prior the correlated markers leave their types' init terms and the
                # 'head' type has none (chmosh.py:362-367); a type left without markers reports 0
                if k == 'head':
                    continue
                mask = mask.copy()
                mask[self.head_ids] = False
            w_init[mask] = wts['init'][k]
            sse[f'init_{k}'] = float(((r_init[mask] * wts['init'][k]) ** 2).sum())
        if self.head_ids is not None:                                                            # chmosh.py:368-369
            r_hc = wts['init_head_corr'] * self.head_corr.dot(r_init[self.head_ids])            # K x 3
            sse['init_head_corr'] = float((r_hc ** 2).sum())
        # betas (AliasedBetas: all shape coefficients of the canonical model, chmosh.py:379)
        if self.free_betas:
            sse['beta'] = float(((self.betas * wts['beta']) ** 2).sum())
        # surface distance of the latent markers (chmosh.py:71-82,380)
        sq, tri, part, d_s, d_t = self.backend.squared_distance(self.ml, can_v, self.faces)
        vn = vertex_normals(can_v, self.faces)
        fv = self.faces[tri]
        tnrm = np.cross(can_v[fv[:, 1]] - can_v[fv[:, 0]], can_v[fv[:, 2]] - can_v[fv[:, 0]])
        tnrm /= np.linalg.norm(tnrm, axis=1, keepdims=True)
        rows = np.arange(M)
        near = np.where((part == 0)[:, None], tnrm, 0.0)
        isv = part > 3
        near[isv] = vn[fv[rows[isv], part[isv] - 4]]
        ise = (part > 0) & (part <= 3)
        near[ise] = vn[fv[rows[ise], part[ise] - 1]] + vn[fv[rows[ise], part[ise] % 3]]
        direction = np.sign((0.5 * d_s * near).sum(1))               # sample - nearest point = 1/2 d(squared distance)/d(sample)
        xs = sq * direction
        dist = np.sqrt(np.abs(xs)) * np.sign(xs)
        r_surf = (dist - self.m2b) * wts['surf']
        sse['surf'] = float((r_surf ** 2).sum())
        total = float(sum(sse.values()))
        if not want_jac:
            return total, sse, dev

        # ---------------- normal equations, unknowns [betas (nb) | latent markers (3M) | frame 0 (n_p) | frame 1 | ...];
        # a frame's private block is [trans | pose ids | expressions (optimize_face, detailed steps)], the free list's order
        ns = nb + 3 * M
        n = ns + F * n_p
        A = np.zeros((n, n))
        g = np.zeros(n)
        Cs = self.can.C                                                                          # V x 3 x nb (free shape block)
        k, Fcan, dk_dv = attachment_coefficients(can_v[pk.closest], self.ml)
        dk_db = np.einsum('mit,mtb->mib', dk_dv, Cs[pk.closest][:, :, :, :nb].reshape(M, 9, nb)) if nb else np.zeros((M, 3, 0))
        for f in range(F):
            Jf = dev['J'][f]                                     # 3M x n_f, weighted, zero rows where invisible
            r = dev['r'][f]
            wv = wts['data'] * self.vis[f].astype(np.float64)
            # the weight of the rows through the attachment; with the robust data term each row also takes the psi' the
            # device applied to its own columns of that row
            wa = wv[:, None, None]
            if self.robust_sigma is not None:
                wa = wa * data_dpsi_gm(r, wts['data'], self.robust_sigma).reshape(M, 3, 1)
            Fp, _, _ = local_frames(dev['vp'][f, 0::3], dev['vp'][f, 1::3], dev['vp'][f, 2::3])   # rows f1, f2, f3 of the posed frames
            FpT = np.transpose(Fp, (0, 2, 1))                     # columns
            Jp = Jf[:, :n_p]
            Jb = Jf[:, n_p:].reshape(M, 3, nb) + wa * np.einsum('mij,mjb->mib', FpT, dk_db)
            Jb = Jb.reshape(3 * M, nb)
            Jm = wa * np.einsum('mij,mjk->mik', FpT, Fcan)                                         # 3x3 blocks d r_i / d ml_i
            c0 = ns + f * n_p
            A[c0:c0 + n_p, c0:c0 + n_p] = dev['A'][f][:n_p, :n_p]
            g[c0:c0 + n_p] = dev['g'][f][:n_p]
            if nb:
                A[:nb, :nb] += Jb.T.dot(Jb)
                Apb = Jp.T.dot(Jb)
                A[c0:c0 + n_p, :nb] = Apb
                A[:nb, c0:c0 + n_p] = Apb.T
                g[:nb] -= Jb.T.dot(r)
            Jp3, r3 = Jp.reshape(M, 3, n_p), r.reshape(M, 3)
            Apm = np.einsum('mip,mik->pmk', Jp3, Jm).reshape(n_p, 3 * M)
            A[c0:c0 + n_p, nb:ns] = Apm
            A[nb:ns, c0:c0 + n_p] = Apm.T
            g[nb:ns] -= np.einsum('mik,mi->mk', Jm, r3).reshape(-1)
            mm = np.einsum('mik,mil->mkl', Jm, Jm)
            for i in range(M):
                A[nb + 3 * i:nb + 3 * i + 3, nb + 3 * i:nb + 3 * i + 3] += mm[i]
            if nb:
                Abm = np.einsum('mib,mik->bmk', Jb.reshape(M, 3, nb), Jm).reshape(nb, 3 * M)
                A[:nb, nb:ns] += Abm
                A[nb:ns, :nb] += Abm.T
        # init rows: d/d ml = w I, d/d betas = -w dinit/dbetas
        w2 = w_init ** 2
        for i in range(M):
            A[nb + 3 * i:nb + 3 * i + 3, nb + 3 * i:nb + 3 * i + 3] += w2[i] * np.eye(3)
        g[nb:ns] -= (w2[:, None] * r_init).reshape(-1)
        if nb:
            Gi = -np.einsum('mit,mtb->mib', dinit_dv, Cs[self.closest0][:, :, :, :nb].reshape(M, 9, nb))      # d r_init / d betas (unweighted)
            A[:nb, :nb] += np.einsum('m,mib,mic->bc', w2, Gi, Gi)
            Abm = np.einsum('m,mib->bmi', w2, Gi).reshape(nb, 3 * M)
            A[:nb, nb:ns] += Abm
            A[nb:ns, :nb] += Abm.T
            g[:nb] -= np.einsum('m,mib,mi->b', w2, Gi, r_init)
            # betas prior
            A[:nb, :nb] += wts['beta'] ** 2 * np.eye(nb)
            g[:nb] -= wts['beta'] ** 2 * self.betas[:nb]
        if self.head_ids is not None:
            # head-marker correlation rows w corr (ml - init)[head_ids]: dense over the latent unknowns of the correlated
            # markers (d/d ml[head_ids[j]] = w corr[:, j] (x) I) and, with a free shape, d/d betas = w corr (x) d r_init/d betas
            wh = wts['init_head_corr']
            Jh = np.zeros((len(self.head_corr), 3, ns))
            for j, i in enumerate(self.head_ids):
                Jh[:, :, nb + 3 * i:nb + 3 * i + 3] += wh * self.head_corr[:, j, None, None] * np.eye(3)
            if nb:
                Jh[:, :, :nb] = wh * np.einsum('kh,hib->kib', self.head_corr, Gi[self.head_ids])
            Jh = Jh.reshape(-1, ns)
            A[:ns, :ns] += Jh.T.dot(Jh)
            g[:ns] -= Jh.T.dot(r_hc.reshape(-1))
        # surf rows
        with np.errstate(divide='ignore', invalid='ignore'):
            gs = np.nan_to_num(0.5 / np.sqrt(np.abs(xs))) * (xs != 0) * direction * wts['surf']
        Js_m = gs[:, None] * d_s                                                                  # M x 3
        for i in range(M):
            A[nb + 3 * i:nb + 3 * i + 3, nb + 3 * i:nb + 3 * i + 3] += np.outer(Js_m[i], Js_m[i])
        g[nb:ns] -= (Js_m * r_surf[:, None]).reshape(-1)
        if nb:
            Js_b = gs[:, None] * np.einsum('mt,mtb->mb', d_t, Cs[fv][:, :, :, :nb].reshape(M, 9, nb))  # M x nb
            A[:nb, :nb] += Js_b.T.dot(Js_b)
            Abm = np.einsum('mb,mk->bmk', Js_b, Js_m).reshape(nb, 3 * M)
            A[:nb, nb:ns] += Abm
            A[nb:ns, :nb] += Abm.T
            g[:nb] -= Js_b.T.dot(r_surf)
        self._last_total = total        # (the dog-leg needs the SSE of the linearisation point)
        return total, sse, dev, A, g, (pk, free, n_p)

    # ---- state <-> unknown vector -------------------------------------------------------------------------------------
    def get_x(self, pose_ids, nb, ne=0):
        parts = [self.betas[:nb], self.ml.reshape(-1)]
        for f in range(self.F):
            parts += [self.trans[f], self.pose[f, pose_ids], self.expr[f, :ne]]
        return np.concatenate(parts)

    def set_x(self, x, pose_ids, nb, ne=0):
        M, npi = self.M, len(pose_ids)
        self.betas[:nb] = x[:nb]
        self.ml = x[nb:nb + 3 * M].reshape(M, 3).copy()
        o = nb + 3 * M
        for f in range(self.F):
            self.trans[f] = x[o:o + 3]
            self.pose[f, pose_ids] = x[o + 3:o + 3 + npi]
            self.expr[f, :ne] = x[o + 3 + npi:o + 3 + npi + ne]
            o += 3 + npi + ne

    # ---- chumpy's dog-leg (SURVEY.md A.6; the control flow of csrc/mosh2_device.cuh solve_frame on dense float64 arrays) --
    def minimize(self, wts, detailed, e_3, maxiter, delta_0=0.5, e_1=1e-15, e_2=1e-15):
        nb = self.nb if self.free_betas else 0
        _, _, _, A, g, (pk, free, n_p) = self.evaluate(True, wts, detailed)[:6]
        pose_ids = np.asarray([int(i) - 3 for i in free[3:n_p] if i < 3 + pk.p_red], dtype=np.int64)
        ne = n_p - 3 - len(pose_ids)                     # the expression columns follow the pose ids (optimize_face, Step 2)
        self._dogleg(A, g, self.get_x(pose_ids, nb, ne), lambda x: self.set_x(x, pose_ids, nb, ne),
                     lambda: self.evaluate(False, wts, detailed)[0], lambda: self.evaluate(True, wts, detailed)[3:5],
                     nb + 3 * self.M, n_p, e_3, maxiter, delta_0, e_1, e_2)

    # ---- extra_initial_rigid_adjustment (chmosh.py:230-232): the unweighted data residual of every picked frame wrt its root
    #      orientation and translation, the latent markers, the shape and the attachment fixed ---------------------------------
    def evaluate_rigid(self, want_jac: bool):
        """Data SSE, and with want_jac the block-diagonal normal equations of the unknowns [trans | pose[:3]] of every frame."""
        F = self.F
        self.stats['evaluations'] += 1
        self.stats['linearisations'] += int(want_jac)
        pk = self.pack_for(False, self.can(self.betas[:self.nb]))
        pk.free_step1 = np.arange(6, dtype=np.int32)                     # columns 0..5 of x = [trans | pose | linear block]
        x = np.zeros((F, pk.nx))
        x[:, :3], x[:, 3:3 + pk.p_red] = self.trans, self.pose
        if self.face:
            x[:, 3 + pk.p_red + pk.n_dmpl - pk.n_expr:] = self.expr
        opts = _lib.make_options(None)
        opts.wt_data, opts.wt_poseB, opts.wt_poseH = 1.0, 0.0, 0.0
        if self.robust_sigma is not None:                   # (rows psi(e): the weight is 1)
            opts.robust_sigma = self.robust_sigma
        dev = self.backend.linearize(pk, opts, self.obs, self.vis, x, 1, want_jac)
        total = float(dev['errs'][:, 0].sum())
        if not want_jac:
            return total
        A = np.zeros((6 * F, 6 * F))
        for f in range(F):
            A[6 * f:6 * f + 6, 6 * f:6 * f + 6] = dev['A'][f]
        self._last_total = total
        return A, dev['g'].reshape(-1).copy()

    def get_rigid_x(self):
        return np.concatenate([self.trans, self.pose[:, :3]], axis=1).reshape(-1)

    def set_rigid_x(self, x):
        x = x.reshape(self.F, 6)
        self.trans[:] = x[:, :3]
        self.pose[:, :3] = x[:, 3:]

    def minimize_rigid(self, maxiter, e_3=1e-3, delta_0=0.5, e_1=1e-15, e_2=1e-15):
        """One dog-leg over all picked frames with one trust region; the normal equations have no shared block."""
        A, g = self.evaluate_rigid(True)
        self._dogleg(A, g, self.get_rigid_x(), self.set_rigid_x, lambda: self.evaluate_rigid(False),
                     lambda: self.evaluate_rigid(True), 0, 6, e_3, maxiter, delta_0, e_1, e_2)

    def _dogleg(self, A, g, p, set_x, sse_at, linearize, ns, n_p, e_3, maxiter, delta_0, e_1, e_2):
        """The dog-leg iterations from the normal equations (A, g) at p, whose SSE is self._last_total.  ``set_x`` puts a
        state vector into the solver, ``sse_at()`` evaluates the objective there, ``linearize()`` returns its (A, g)."""
        sse0 = self._last_total
        delta = delta_0
        done = np.linalg.norm(g, np.inf) < e_1
        it = 0
        while not done:
            it += 1
            self.stats['iterations'] += 1
            Ag = A.dot(g)
            d_sd = (g.dot(g) / g.dot(Ag)) * g
            d_gn = None
            while True:
                if np.linalg.norm(d_sd) >= delta:
                    d_dl = (delta / np.linalg.norm(d_sd)) * d_sd
                else:
                    if d_gn is None:
                        d_gn = _solve_arrow(A, g, ns, n_p, self.F)
                    if np.linalg.norm(d_gn) <= delta:
                        d_dl = d_gn.copy()
                    else:
                        dsq = delta ** 2
                        diff = d_gn - d_sd
                        sd2 = d_sd.dot(d_sd)
                        pnow = diff.dot(diff) * dsq + d_gn.dot(d_sd) ** 2 - d_gn.dot(d_gn) * sd2
                        d_dl = d_sd + (dsq - sd2) / (diff.dot(d_sd) + np.sqrt(pnow)) * diff
                improved = False
                if np.linalg.norm(d_dl) <= e_2 * np.linalg.norm(p):
                    done = True
                else:
                    set_x(p + d_dl)
                    sse1 = sse_at()
                    rho = sse0 - sse1
                    if rho > 0:
                        with np.errstate(divide='ignore', invalid='ignore'):
                            rho = rho / (2.0 * g.dot(d_dl) - d_dl.dot(A.dot(d_dl)))
                    improved = rho > 0
                    if improved:
                        p = p + d_dl
                        if e_3 > 0.0 and (sse0 - sse1) / sse0 < e_3:
                            done = True
                        else:
                            A, g = linearize()
                            sse0 = sse1
                            if np.linalg.norm(g, np.inf) < e_1:
                                done = True
                    if rho > 0.9:
                        delta = max(delta, 2.5 * np.linalg.norm(d_dl))
                    elif rho < 0.05:
                        delta *= 0.25
                    if delta <= e_2 * np.linalg.norm(p):
                        done = True
                if done or improved:
                    break
            if not done and it >= maxiter:
                done = True
        set_x(p)
        self.stats['minimisations'] += 1

    def run(self):
        cfg = self.cfg
        extra_rigid = bool(_get(cfg.opt_settings, 'extra_initial_rigid_adjustment', False))
        if extra_rigid and not self.reference_options:                                           # chmosh.py:230-232
            raise NotImplementedError('opt_settings.extra_initial_rigid_adjustment runs only when asked to '
                                      '(reference_options=True)')
        ann = list(cfg.opt_settings.weights['stagei_wt_annealing'])
        # rigid alignment of every frame to its markers (chmosh.py:225-229)
        _, _, dev = self.evaluate(False, self.weights_for(ann[0]), False)
        for f in range(self.F):
            v = self.vis[f]
            self.pose[f, :3], self.trans[f] = rigid_fit(dev['markers_sim'][f][v], self.obs[f][v])
        if extra_rigid:     # (e_3 is the reference's fixed 1e-3, not stagei_lr)
            self.minimize_rigid(int(cfg.opt_settings.maxiter))
        sse = {}
        for tidx, a in enumerate(ann):
            detailed = tidx > len(ann) - 3                                                       # chmosh.py:311
            wts = self.weights_for(a)
            self.minimize(wts, detailed, float(cfg.opt_settings.stagei_lr), int(cfg.opt_settings.maxiter))
            _, sse, dev = self.evaluate(False, wts, detailed)
        return sse, dev


def mosh_stagei(stagei_frames: List[Dict[str, np.ndarray]], cfg, betas_fname=None, v_template_fname=None, *, marker_meta=None,
                device: int = 0, backend=None, face_with_free_shape: bool = False, reference_options: bool = False,
                robust_data_sigma: Optional[float] = None) -> dict:
    """Stage I of MoSh++ on one H100.  Positional arguments as in the reference (chmosh.py:83-85).  The marker layout is read
    from ``cfg.dirs.marker_layout.fname`` like the reference does (chmosh.py:120-125), or handed over loaded as ``marker_meta``.

    ``face_with_free_shape``: with ``optimize_betas`` and ``optimize_face`` on SMPL-X, fit the shape and the jaw and expressions
    of every picked frame together instead of raising NotImplementedError (the reference's answer; its log suggests running
    Stage I twice, for the shape without the face markers and then for the face with that shape).  Off by default.

    ``reference_options``: honour ``moshpp.head_marker_corr_fname`` (the head-marker correlation prior, chmosh.py:252-266,
    360-373) and ``opt_settings.extra_initial_rigid_adjustment`` (chmosh.py:230-232) as the reference does.  Off by default:
    then either option in ``cfg`` raises NotImplementedError.  With both options off in ``cfg`` the keyword changes nothing.

    ``robust_data_sigma``: None (default) = the reference's least-squares data term; sigma > 0 (metres) = the Geman-McClure
    data term of Stage II (``chmosh.mosh_stageii``): every data row of the annealing steps and of the extra rigid adjustment
    is wd sigma e / sqrt(sigma^2 + e^2) per coordinate of a visible marker's residual e = sim - obs, so that a swapped label or
    a ghost marker in the picked frames pulls the shape and the latent markers with a bounded force.  The per-frame
    Procrustes start and the init, head-correlation, shape, surface and pose terms stay least squares.
    ``stagei_errs['data']`` then reports the robust SSE, the value minimised, and sigma is recorded in
    ``stagei_debug_details['b200']['robust_data_sigma']`` (absent without it).  A sigma <= 0 or a non-finite one raises
    ValueError."""
    check_robust_sigma(robust_data_sigma)
    if marker_meta is None:                                                                      # chmosh.py:120-125
        mc = cfg.mocap
        marker_meta = load_marker_layout(cfg.dirs.marker_layout.fname, exclude_markers=_get(mc, 'exclude_markers'),
                                         exclude_marker_types=_get(mc, 'exclude_marker_types'), only_markers=_get(mc, 'only_markers'))
    if marker_meta.get('surface_model_type', cfg.surface_model.type) != cfg.surface_model.type:
        raise ValueError(f"marker layout surface_model_type doesnt match that of curent mosh session surface_model.type: "
                         f"{marker_meta['surface_model_type']} == {cfg.surface_model.type}")
    betas = None
    if betas_fname is not None:
        assert str(betas_fname).endswith('.npz'), ValueError(f'invalid numpy betas_fname: {betas_fname}')
        betas = np.load(betas_fname)['betas']
    v_template = _read_vertices(v_template_fname) if v_template_fname else None
    s = StageI(stagei_frames, cfg, marker_meta, betas=betas, v_template=v_template, backend=backend or DeviceBackend(device),
               face_with_free_shape=face_with_free_shape, reference_options=reference_options,
               robust_data_sigma=robust_data_sigma)
    sse, dev = s.run()
    can_v = s.can(s.betas[:s.nb])
    d2 = ((s.ml[:, None, :] - can_v[None]) ** 2).sum(-1)                                        # chmosh.py:422-424: nearest vertex
    vids = d2.argmin(1)
    sims_all = [dev['markers_sim'][f].copy() for f in range(s.F)]
    labels_obs = [[l for l, v in zip(s.labels, s.vis[f]) if v] for f in range(s.F)]
    dbg = {'opt_models_trans': [t.copy() for t in s.trans], 'opt_models_pose': [p.copy() for p in s.pose], 'stagei_errs': sse,
           'stagei_markers_sim_all': sims_all, 'stagei_markers_sim': [sims_all[f][s.vis[f]] for f in range(s.F)],
           'stagei_markers_obs': [s.obs[f][s.vis[f]] for f in range(s.F)], 'stagei_labels_obs': labels_obs,
           'b200': dict(s.stats)}
    if s.robust_sigma is not None:
        dbg['b200']['robust_data_sigma'] = s.robust_sigma
    if s.face:
        dbg['opt_models_expression'] = [e.copy() for e in s.expr]    # betas[es:es + ne] of each picked frame's model
    out = {'betas': s.betas.copy(), 'markers_latent': s.ml.copy(), 'latent_labels': s.labels, 'marker_meta': marker_meta,
           'markers_latent_vids': {l: int(v) for l, v in zip(s.labels, vids)}, 'stagei_debug_details': dbg}
    if v_template_fname is not None:
        out['v_template_fname'] = v_template_fname
        dbg['v_template'] = s.model.v_template.copy()
    return out
