"""Stage I of MoSh++ in float64 numpy (oracle; test infrastructure only -- PARITY UNPINNED, see below).

Restates chmosh.py:83-455 ``mosh_stagei``: shape (betas), latent marker positions and the poses / translations of the
(usually twelve) picked frames, estimated jointly by four annealed ``ch.minimize(method='dogleg')`` calls over

    data   (obs - sim) * wt_data                       chmosh.py:202-213,350     sim = TransformedLms(TransformedCoeffs(can, ML), posed)
    poseB  prior(pose[body]) * wt_poseB   per frame    353-356                   (+ poseB_jangles for the horse, 358-360)
    init_k (ML - init(betas))[type k] * wt_init_k      362,376-377               init rides on the canonical body (185-186)
    beta   betas * wt_beta                             379                       AliasedBetas = all betas of the canonical model
    surf   (signed distance(ML, can mesh) - m2b) * wt_surf   380, 57-82          PtsToMesh(signed, rho = identity, not normalised)
    poseH  pose[fingers] * wt_poseH       per frame    395-397                   last two annealing steps only

with free variables trans, ML, pose[pose_ids] of every frame and betas[:num_betas] (389-407).  The marker attachment
(8-NN local frames on the canonical body, transformed_lm.py:59-113) is re-made whenever ML or betas change, exactly as
``TransformedCoeffs.on_changed`` does; its derivatives are those chumpy forms through ``_result`` (the neighbour ids are
constants of an evaluation).

Built on lbs.py / markers.py / prior.py / rigid.py / dogleg.py / mesh_distance.py.  What cannot be pinned here, on top of
chumpy's dog-leg and psbody.smpl's LBS (oracle/__init__.py): psbody.mesh's ``estimate_vertex_normals`` and AABB-tree
nearest-part query (restated as area-weighted vertex normals and a brute-force closest-point search), and the order in
which chumpy stacks the residual blocks (irrelevant to J^T J).

The keywords of the product's ``mosh_stagei``, on the one solver:
  * ``moshpp.optimize_face`` (SMPL-X): every frame's jaw and expressions, free in the two detailed steps with their poseF /
    expr terms (chmosh.py:136-151,163-170,283-297,322-324,396-401); with a free shape the reference raises (287-291),
    ``face_with_free_shape=True`` fits the shape and the expressions together;
  * ``reference_options=True``: the head-marker correlation prior (``init_head_corr``, chmosh.py:252-266,360-373) and the
    extra initial rigid adjustment (230-232); without it the prior is not applied and the adjustment raises
    NotImplementedError when the solver runs;
  * ``robust_data_sigma``: the Geman-McClure data term (robust.py) in the annealing steps and the extra rigid adjustment.
The dog (``animal_dog``) is a model type like the others: its max-mixture prior and pose ids are prior.py's.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
from sklearn.neighbors import NearestNeighbors

from . import mesh_distance as md
from .dogleg import minimize_dogleg
from .lbs import LBS, OracleModel
from .markers import TransformedCoeffs, _N, _skew, nrm, transformed_lms
from .prior import DOG_POSE_IDS, HORSE_JANGLES_IDS, HORSE_JANGLES_SIGNS, create_body_prior, horse_joint_angles
from .rigid import perform_rigid_adjustment
from .robust import gm_dpsi, gm_psi

NUM_TRAIN_MARKERS = 46   # chmosh.py:100


def vertex_normals(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """Normalised sum of the area-scaled triangle normals around every vertex (scan2mesh/ch_vert_normals.py:86-139)."""
    tn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    vn = np.zeros_like(v)
    for k in range(3):
        np.add.at(vn, f[:, k], tn)
    ss = (vn ** 2).sum(1)
    ss[ss == 0] = 1e-10
    return vn / np.sqrt(ss)[:, None]


def coeff_jacobians(can_tri: np.ndarray, ml: np.ndarray):
    """k = F^T (ml - v0) of one marker on its canonical triple (3 x 3 rows v0, v1, v2): (k, dk/dml 3x3, dk/d(v0,v1,v2) 3x9)."""
    v0, v1, v2 = can_tri
    e1, e2 = v1 - v0, v2 - v0
    n = np.cross(e1, e2)
    f1 = e1 / np.linalg.norm(e1)
    f2 = n / np.linalg.norm(n)
    f3 = np.cross(f1, f2)
    d = ml - v0
    F = np.stack([f1, f2, f3])                      # rows
    k = F.dot(d)
    df1_de1 = _N(e1)
    df2_de1 = _N(n).dot(-_skew(e2))
    df2_de2 = _N(n).dot(_skew(e1))
    df3_de1 = -_skew(f2).dot(df1_de1) + _skew(f1).dot(df2_de1)
    df3_de2 = _skew(f1).dot(df2_de2)
    dk_de1 = np.stack([d.dot(df1_de1), d.dot(df2_de1), d.dot(df3_de1)])
    dk_de2 = np.stack([np.zeros(3), d.dot(df2_de2), d.dot(df3_de2)])
    dk_dv = np.zeros((3, 9))
    dk_dv[:, 0:3] = -F - dk_de1 - dk_de2
    dk_dv[:, 3:6] = dk_de1
    dk_dv[:, 6:9] = dk_de2
    return k, F, dk_dv


def signed_surface_distance(samples, verts, faces, vn=None, want_jac=False):
    """PtsToMesh(signed=True, rho=identity, normalize=False) (mesh_distance_main.py:160-183,215-300): sign * sqrt(squared
    distance to the nearest triangle part), sign = side of the (face / summed vertex) normal of that part.
    Returns d [S] and, if want_jac, (d_sample [S,3], tri [S], d_tri [S,9])."""
    r, Ds, Dt, tri, part = md.somedistance(samples, verts, faces, kind=md.KIND_SQUARED)
    if vn is None:
        vn = vertex_normals(verts, faces)
    fv = faces[tri]
    a, b, c = verts[fv[:, 0]], verts[fv[:, 1]], verts[fv[:, 2]]
    near_n = np.zeros_like(samples)
    nearest_point = np.zeros_like(samples)
    for s in range(len(samples)):
        p = int(part[s])
        if p == 0:
            near_n[s] = nrm(np.cross(b[s] - a[s], c[s] - a[s])[None])[0]
        elif p > 3:
            near_n[s] = vn[fv[s, p - 4]]
        else:
            near_n[s] = vn[fv[s, p - 1]] + vn[fv[s, p % 3]]
    # diff = sample - nearest point = -1/2 d(squared distance)/d(sample) * (-1): the gradient of |x - c|^2 wrt x is 2 (x - c)
    diff = 0.5 * Ds
    direction = np.sign((diff * near_n).sum(1))
    sq = r
    d = np.sqrt(np.abs(sq * direction)) * np.sign(sq * direction)
    if not want_jac:
        return d
    with np.errstate(divide='ignore', invalid='ignore'):
        g = np.nan_to_num(0.5 / np.sqrt(np.abs(sq * direction))) * (sq * direction != 0)
    return d, (g * direction)[:, None] * Ds, tri, (g * direction)[:, None] * Dt


class StageISolver:
    """The chumpy graph of chmosh.py:83-455 as explicit state + residual / Jacobian evaluation, with the keywords of the
    product's ``mosh_stagei`` (see ``mosh_stagei`` below)."""

    def __init__(self, stagei_frames: List[Dict[str, np.ndarray]], cfg, marker_meta, betas=None, v_template=None, *,
                 face_with_free_shape=False, reference_options=False, robust_data_sigma=None):
        sm, mp = cfg.surface_model, cfg.moshpp
        self.cfg = cfg
        self.marker_meta = marker_meta
        self.latent_labels = list(marker_meta['marker_vids'].keys())
        M = self.n_markers = len(self.latent_labels)
        F = self.n_frames = len(stagei_frames)
        avail_labels = set(k for fr in stagei_frames for k in fr.keys())
        self.optimize_fingers = bool(mp.optimize_fingers)
        if self.optimize_fingers:                                                               # chmosh.py:130-141
            if not np.any(['finger' in m for m in marker_meta['marker_type_mask'].keys()]):
                self.optimize_fingers = False
            elif not np.any([('finger' in t) and l in avail_labels for l, t in marker_meta['marker_type'].items()]):
                self.optimize_fingers = False
        self.optimize_betas = bool(mp.optimize_betas)
        # optimize_face: off with a free shape when the face markers are excluded (chmosh.py:103-118), off without a face-type
        # marker in the layout or a face label in the frames (127-137); only SMPL-X has a jaw and expression components; with a
        # free shape the reference raises when it runs (287-291), face_with_free_shape fits the shape and the expressions together
        self.face = bool(mp.get('optimize_face', False)) and sm.type == 'smplx'
        if self.face and self.optimize_betas and 'face' in (cfg.mocap.get('exclude_marker_types') or []):
            self.face = False
        if self.face and not np.any(['face' in t for t in marker_meta['marker_type_mask'].keys()]):
            self.face = False
        if self.face and not np.any([('face' in t) and l in avail_labels for l, t in marker_meta['marker_type'].items()]):
            self.face = False
        self.face_with_free_shape = face_with_free_shape
        # every frame's model: the shape plus the frame's expressions at betas[betas_expr_start_id:][:num_expressions]; the
        # canonical body keeps zero expressions
        self.face_ids = [66, 67, 68] if self.face else []                                       # the jaw (line 293)
        es = int(sm.betas_expr_start_id) if self.face else 0
        self.expr_ids = np.arange(es, es + (int(sm.num_expressions) if self.face else 0))
        self.expr = np.zeros((F, len(self.expr_ids)))
        self.robust_sigma = robust_data_sigma           # None: the reference's least-squares data term
        # reference_options: the head-marker correlation prior (chmosh.py:252-266; corr_ids / corr stay None when it does not
        # apply) and the extra rigid adjustment (230-232, in run)
        self.reference_options = reference_options
        self.corr_ids, self.corr = None, None
        corr_fname = mp.get('head_marker_corr_fname') if reference_options else None
        if corr_fname is not None:
            head = np.load(corr_fname)
            if all(l in marker_meta['marker_vids'] for l in head['mrk_labels']):
                self.corr_ids = [self.latent_labels.index(l) for l in head['mrk_labels']]
                self.corr = np.asarray(head['corr'], dtype=np.float64)
        self.model = m = OracleModel(sm.fname, pose_hand_prior_fname=mp.pose_hand_prior_fname, use_hands_mean=sm.use_hands_mean,
                                     dof_per_hand=sm.dof_per_hand, v_template=v_template, surface_model_type=sm.type)
        with open(sm.fname, 'rb') as f:
            import pickle
            self.faces = np.asarray(pickle.load(f, encoding='latin-1')['f'], dtype=np.int64)
        self.prior = create_body_prior(m.model_type, mp.pose_body_prior_fname)
        self.nb = int(sm.num_betas)
        self.betas = np.zeros(m.n_betas_model)
        if betas is not None:
            self.betas[:self.nb] = np.asarray(betas)[:self.nb]                                  # chmosh.py:169-172
        self.pose = np.zeros((F, m.pose_size))
        self.trans = np.zeros((F, 3))
        self.full_lbs = LBS(m, None)
        # d can_v / d betas[:nb]: NOT the shape directions where the canonical pose is not the rest pose (use_hands_mean: the
        # hands of can_model are in their mean pose, smpl_fast_derivatives.py:194-204); can_v is affine in betas (rotations fixed)
        _, _, self.Sdirs = self.full_lbs(np.zeros(m.pose_size), self.betas, np.zeros(3), True, beta_ids=np.arange(self.nb))

        # prepare_mosh_markers_latent, chmosh.py:57-82
        can_v = self.can_v()
        vn = vertex_normals(can_v, self.faces)
        self.m2b = np.ones(M) * 0.0095
        for mask_type, mask in marker_meta['marker_type_mask'].items():
            self.m2b[np.asarray(mask)] = marker_meta['m2b_distance'][mask_type]
        vids = np.asarray(list(marker_meta['marker_vids'].values()), dtype=np.int64)
        self.ml = can_v[vids] + vn[vids] * self.m2b[:, None]
        self.tc0 = TransformedCoeffs(can_v, self.ml)                                            # tc2: constants (185)

        # observed markers per frame (chmosh.py:193-206; the order inside a frame does not enter the objective)
        self.obs, self.lm_ids, self.labels_obs = [], [], []
        for fr in stagei_frames:
            labs = [l for l in self.latent_labels if l in fr and not np.any(np.isnan(fr[l]))]
            self.labels_obs.append(labs)
            self.lm_ids.append(np.asarray([self.latent_labels.index(l) for l in labs], dtype=np.int64))
            self.obs.append(np.vstack([fr[l] for l in labs]))

        all_ids = list(range(m.pose_size))                                                      # chmosh.py:268-309
        self.root_ids, self.body_ids, self.finger_ids = all_ids[:3], [], []
        if sm.type == 'smpl':
            self.body_ids = all_ids[3:]
        elif sm.type == 'smplh':
            self.body_ids = all_ids[3:66]
            if self.optimize_fingers:
                self.finger_ids = all_ids[66:]
        elif sm.type == 'smplx':
            self.body_ids = all_ids[3:66]
            if self.optimize_fingers:
                self.finger_ids = all_ids[75:]
        elif sm.type == 'mano':
            self.finger_ids = all_ids[3:]
        elif sm.type == 'animal_horse':
            self.body_ids = all_ids[3:84]
        elif sm.type == 'animal_dog':
            self.body_ids = [all_ids[i] for i in DOG_POSE_IDS]
        else:
            raise NotImplementedError(sm.type)
        self.stats = dict(r_evals=0, j_evals=0, iterations=0, minimizations=0)

    # ---------------------------------------------------------------------------------------------------------------
    def can_v(self):
        return self.full_lbs(np.zeros(self.model.pose_size), self.betas, np.zeros(3))

    def frame_betas(self, f):
        b = self.betas.copy()
        b[self.expr_ids] = self.expr[f]
        return b

    def pose_ids_for(self, detailed: bool):
        ids = self.root_ids + self.body_ids
        if len(self.body_ids) and not self.cfg.moshpp.optimize_toes:
            ids = list(set(ids).difference(set(range(30, 36))))                                 # chmosh.py:389-390
        if detailed:
            ids = ids + (self.finger_ids if self.optimize_fingers else []) + self.face_ids      # chmosh.py:392-402
        return np.asarray(sorted(set(ids)), dtype=np.int64)

    def markers_sim_all(self):
        can_v = self.can_v()
        tc = TransformedCoeffs(can_v, self.ml)
        lbs = LBS(self.model, tc.closest[:, :3].reshape(-1))
        out = []
        for f in range(self.n_frames):
            v = lbs(self.pose[f], self.frame_betas(f), self.trans[f]).reshape(-1, 3, 3)
            out.append(transformed_lms(tc, v[:, 0], v[:, 1], v[:, 2]))
        return out

    def rigid_adjust(self):
        """chmosh.py:225-229."""
        sims = self.markers_sim_all()
        for f in range(self.n_frames):
            rv, T = perform_rigid_adjustment(sims[f][self.lm_ids[f]], self.obs[f])
            self.pose[f, :3] = rv
            self.trans[f] = T

    def rigid_residual(self, xr, want_jac):
        """The objective of the extra rigid adjustment (chmosh.py:231): the data rows at weight 1 (robust with
        robust_data_sigma) wrt xr = [trans | pose[:3]] of every frame, the rest fixed."""
        fr = xr.reshape(self.n_frames, 6)
        self.trans[:], self.pose[:, :3] = fr[:, :3], fr[:, 3:]
        pose_ids = np.arange(3)
        off = self.layout(pose_ids, False)[2]
        rows = list(self.data_rows(want_jac, pose_ids, False, False, 1.0, self.can_v()))
        r = np.concatenate([a for a, _ in rows])
        return (r, np.vstack([J for _, J in rows])[:, off:]) if want_jac else r

    def extra_rigid_adjust(self):
        """chmosh.py:230-232: one dog-leg over every frame's translation and root orientation."""
        x0 = np.hstack([self.trans, self.pose[:, :3]]).reshape(-1)
        xr, st = minimize_dogleg(self.rigid_residual, x0, e_3=1e-3, delta_0=0.5, maxiter=int(self.cfg.opt_settings.maxiter))
        fr = xr.reshape(self.n_frames, 6)
        self.trans[:], self.pose[:, :3] = fr[:, :3], fr[:, 3:]
        self._count(st)

    # ---- residual vector and Jacobian for one annealing step ---------------------------------------------------
    def layout(self, pose_ids, free_betas, free_expr=False):
        """The unknowns [betas[:nb] if free_betas | latent markers (3 M) | frame 0 | frame 1 | ...], a frame's block
        [trans | pose[pose_ids] | expressions if free_expr (the face, detailed steps)]: (nb free, latent-marker offset, frame
        offset, frame block size, total)."""
        nb = self.nb if free_betas else 0
        off_fr = nb + 3 * self.n_markers
        per = 3 + len(pose_ids) + (len(self.expr_ids) if free_expr else 0)
        return nb, nb, off_fr, per, off_fr + self.n_frames * per

    def get_x(self, pose_ids, free_betas, free_expr=False):
        nb, off_ml, off_fr, per, n = self.layout(pose_ids, free_betas, free_expr)
        npi = len(pose_ids)
        x = np.zeros(n)
        x[:nb] = self.betas[:nb]
        x[off_ml:off_fr] = self.ml.reshape(-1)
        fr = x[off_fr:].reshape(self.n_frames, per)
        fr[:, :3] = self.trans
        fr[:, 3:3 + npi] = self.pose[:, pose_ids]
        fr[:, 3 + npi:] = self.expr[:, :per - 3 - npi]
        return x

    def set_x(self, x, pose_ids, free_betas, free_expr=False):
        nb, off_ml, off_fr, per, n = self.layout(pose_ids, free_betas, free_expr)
        npi = len(pose_ids)
        self.betas[:nb] = x[:nb]
        self.ml = x[off_ml:off_fr].reshape(-1, 3).copy()
        fr = x[off_fr:].reshape(self.n_frames, per)
        self.trans[:] = fr[:, :3]
        self.pose[:, pose_ids] = fr[:, 3:3 + npi]
        self.expr[:, :per - 3 - npi] = fr[:, 3 + npi:]

    def data_rows(self, want_jac, pose_ids, free_betas, free_expr, wd, can_v):
        """The data rows of every frame (chmosh.py:202-213,349), (obs - sim) wd or with robust_data_sigma wd psi(obs - sim),
        each frame posed on its own betas: yields (r, J or None) per frame.  The shape columns come through the frame's model
        and the marker attachment, the expression columns through the posed vertices only."""
        nbf, off_ml, off_fr, per, n = self.layout(pose_ids, free_betas, free_expr)
        M, npi = self.n_markers, len(pose_ids)
        tc = TransformedCoeffs(can_v, self.ml)                  # transformed_lm.py:59-113, re-made on every change
        tri = tc.closest[:, :3]
        if want_jac:
            Fcan = np.zeros((M, 3, 3))
            dk_db = np.zeros((M, 3, nbf))
            for i in range(M):
                _, Fcan[i], dk_dv = coeff_jacobians(can_v[tri[i]], self.ml[i])
                if nbf:
                    for t in range(3):
                        dk_db[i] += dk_dv[:, 3 * t:3 * t + 3].dot(self.Sdirs[tri[i, t]][:, :nbf])
        bids = np.concatenate([np.arange(nbf), self.expr_ids[:per - 3 - npi]])
        lbs = LBS(self.model, tri.reshape(-1))
        for f in range(self.n_frames):
            ids = self.lm_ids[f]
            res = lbs(self.pose[f], self.frame_betas(f), self.trans[f], want_jac, beta_ids=bids)
            verts = (res[0] if want_jac else res).reshape(M, 3, 3)
            if want_jac:
                sim, loc = transformed_lms(tc, verts[:, 0], verts[:, 1], verts[:, 2], True)
            else:
                sim = transformed_lms(tc, verts[:, 0], verts[:, 1], verts[:, 2])
            e = (self.obs[f] - sim[ids]).reshape(-1)
            r = wd * e if self.robust_sigma is None else wd * gm_psi(e, self.robust_sigma)
            if not want_jac:
                yield r, None
                continue
            dv_pose = res[1].reshape(M, 3, 3, -1)
            dv_beta = res[2].reshape(M, 3, 3, -1)
            J = np.zeros((len(ids), 3, n))
            c0 = off_fr + f * per
            for row, i in enumerate(ids):
                e1, e2 = verts[i, 1] - verts[i, 0], verts[i, 2] - verts[i, 0]
                f1 = e1 / np.linalg.norm(e1)
                nn = np.cross(e1, e2)
                f2 = nn / np.linalg.norm(nn)
                Fp = np.stack([f1, f2, np.cross(f1, f2)], axis=1)             # columns: posed frame
                dpose = sum(loc[i, :, 3 * t:3 * t + 3].dot(dv_pose[i, t]) for t in range(3))
                db = sum(loc[i, :, 3 * t:3 * t + 3].dot(dv_beta[i, t]) for t in range(3))
                J[row, :, c0:c0 + 3] = np.eye(3)
                J[row, :, c0 + 3:c0 + 3 + npi] = dpose[:, pose_ids]
                J[row, :, c0 + 3 + npi:c0 + per] = db[:, nbf:]
                J[row, :, off_ml + 3 * i:off_ml + 3 * i + 3] = Fp.dot(Fcan[i])
                if nbf:
                    J[row, :, :nbf] = db[:, :nbf] + Fp.dot(dk_db[i])
            J = -J.reshape(-1, n) * wd
            if self.robust_sigma is not None:
                J *= gm_dpsi(e, self.robust_sigma)[:, None]
            yield r, J

    def residual(self, x, want_jac, pose_ids, free_betas, wts, detailed, per_term=None, *, free_expr=False, rows=None):
        """r(x) and, if want_jac, J(x) at the unknowns ``x`` of ``layout``; the poseF / expr terms come with free_expr.
        ``per_term`` collects every term's SSE, ``rows`` its rows (a slice of r)."""
        self.set_x(x, pose_ids, free_betas, free_expr)
        nbf, off_ml, off_fr, per, n = self.layout(pose_ids, free_betas, free_expr)
        M, F = self.n_markers, self.n_frames
        m = self.model
        can_v = self.can_v()
        rs, Js = [], []

        def block(name, r, J=None):
            if rows is not None:
                end = sum(len(a) for a in rs) + len(r)
                rows[name] = slice(rows[name].start if name in rows else end - len(r), end)
            rs.append(r)
            if per_term is not None:
                per_term[name] = per_term.get(name, 0.0) + float((r ** 2).sum())
            if want_jac:
                Js.append(J)

        # ---- data
        for r, J in self.data_rows(want_jac, pose_ids, free_betas, free_expr, wts['data'], can_v):
            block('data', r, J)
        # ---- pose prior(s)
        col = {pid: c for c, pid in enumerate(pose_ids)}
        if len(self.body_ids) and self.prior is not None:
            for f in range(F):
                xb = self.pose[f, self.body_ids]
                r = self.prior.r(xb) * wts['poseB']
                J = None
                if want_jac:
                    Jp = self.prior.dr_wrt_x(xb) * wts['poseB']
                    J = np.zeros((r.size, n))
                    for bi, pid in enumerate(self.body_ids):
                        if pid in col:
                            J[:, off_fr + f * per + 3 + col[pid]] = Jp[:, bi]
                block('poseB', r, J)
            if m.model_type == 'animal_horse':
                for f in range(F):
                    xb = self.pose[f, self.body_ids]
                    r = horse_joint_angles(xb) * wts['poseB'] * 2.
                    J = None
                    if want_jac:
                        J = np.zeros((r.size, n))
                        for ri, (bi, sg) in enumerate(zip(HORSE_JANGLES_IDS, HORSE_JANGLES_SIGNS)):
                            pid = self.body_ids[bi]
                            if pid in col:
                                J[ri, off_fr + f * per + 3 + col[pid]] = 2.0 * sg * r[ri]
                    block('poseB_jangles', r, J)
        # ---- init: latent markers against the initial guess riding on the current canonical body (chmosh.py:360-373); with
        #      the head-marker correlation prior the types other than 'head' without the correlated markers, then init_head_corr
        t0 = self.tc0.closest[:, :3]
        if want_jac:
            init, loc0 = transformed_lms(self.tc0, can_v[t0[:, 0]], can_v[t0[:, 1]], can_v[t0[:, 2]], True)
        else:
            init = transformed_lms(self.tc0, can_v[t0[:, 0]], can_v[t0[:, 1]], can_v[t0[:, 2]])
        diff = self.ml - init

        def dinit_db(i):
            return sum(loc0[i, :, 3 * t:3 * t + 3].dot(self.Sdirs[t0[i, t]][:, :nbf]) for t in range(3))
        for k, mask in self.marker_meta['marker_type_mask'].items():
            ids = np.flatnonzero(np.asarray(mask, dtype=bool))
            if self.corr_ids is not None:
                if k == 'head':
                    continue
                ids = np.setdiff1d(ids, self.corr_ids)
            r = (diff[ids] * wts['init'][k]).reshape(-1)
            J = None
            if want_jac:
                J = np.zeros((len(ids), 3, n))
                for row, i in enumerate(ids):
                    J[row, :, off_ml + 3 * i:off_ml + 3 * i + 3] = np.eye(3)
                    if nbf:
                        J[row, :, :nbf] = -dinit_db(i)
                J = J.reshape(-1, n) * wts['init'][k]
            block(f'init_{k}', r, J)
        if self.corr_ids is not None:
            w, C = wts['head_corr'], self.corr
            J = None
            if want_jac:
                J = np.zeros((len(C), 3, n))
                for j, i in enumerate(self.corr_ids):
                    for q in range(len(C)):
                        J[q, :, off_ml + 3 * i:off_ml + 3 * i + 3] += C[q, j] * np.eye(3)
                        if nbf:
                            J[q, :, :nbf] -= C[q, j] * dinit_db(i)
                J = J.reshape(-1, n) * w
            block('init_head_corr', (C.dot(diff[self.corr_ids]) * w).reshape(-1), J)
        # ---- betas
        if free_betas:
            J = None
            if want_jac:
                J = np.zeros((len(self.betas), n))
                J[:nbf, :nbf] = np.eye(nbf) * wts['beta']
            block('beta', self.betas * wts['beta'], J)
        # ---- surface distance of the latent markers
        if want_jac:
            d, d_s, stri, d_t = signed_surface_distance(self.ml, can_v, self.faces, want_jac=True)
            J = np.zeros((M, n))
            for i in range(M):
                J[i, off_ml + 3 * i:off_ml + 3 * i + 3] = d_s[i]
                if nbf:
                    for t in range(3):
                        J[i, :nbf] += d_t[i, 3 * t:3 * t + 3].dot(self.Sdirs[self.faces[stri[i], t]][:, :nbf])
            block('surf', (d - self.m2b) * wts['surf'], J * wts['surf'])
        else:
            block('surf', (signed_surface_distance(self.ml, can_v, self.faces) - self.m2b) * wts['surf'])
        # ---- fingers, then the jaw and the expressions of every frame (detailed steps)
        if detailed and self.optimize_fingers:
            for f in range(F):
                r = self.pose[f, self.finger_ids] * wts['poseH']
                J = None
                if want_jac:
                    J = np.zeros((r.size, n))
                    for ri, pid in enumerate(self.finger_ids):
                        if pid in col:
                            J[ri, off_fr + f * per + 3 + col[pid]] = wts['poseH']
                block('poseH', r, J)
        if free_expr:
            for name in ('poseF', 'expr'):
                for f in range(F):
                    c0 = off_fr + f * per
                    if name == 'poseF':
                        r, cols = self.pose[f, self.face_ids] * wts[name], [c0 + 3 + col[p] for p in self.face_ids]
                    else:
                        r, cols = self.expr[f] * wts[name], list(range(c0 + 3 + len(pose_ids), c0 + per))
                    J = None
                    if want_jac:
                        J = np.zeros((r.size, n))
                        J[np.arange(r.size), cols] = wts[name]
                    block(name, r, J)
        r = np.concatenate(rs)
        if want_jac:
            return r, np.vstack(Js)
        return r

    # ---------------------------------------------------------------------------------------------------------------
    def weights_for(self, anneal):
        w = self.cfg.opt_settings.weights
        out = {'poseB': w['stagei_wt_poseB'] * anneal, 'poseH': w['stagei_wt_poseH'] * anneal, 'beta': w['stagei_wt_betas'] * anneal,
               'data': (w['stagei_wt_data'] / anneal) * (NUM_TRAIN_MARKERS / self.n_markers), 'surf': w['stagei_wt_surf']}
        out['init'] = {}
        for k in self.marker_meta['marker_type_mask'].keys():
            try:
                base = w[f'stagei_wt_init_{k}']
            except (KeyError, AttributeError):
                base = w['stagei_wt_init']
            out['init'][k] = base * anneal
        if self.face:                                                                           # chmosh.py:322-324
            out['poseF'], out['expr'] = w['stagei_wt_poseF'] * anneal, w['stagei_wt_expr'] * anneal
        if self.corr_ids is not None:                                                           # chmosh.py:368-369
            out['head_corr'] = out['init'].get('body', w['stagei_wt_init'] * anneal)
        return out

    def _count(self, st):
        self.stats['r_evals'] += st.r_evals
        self.stats['j_evals'] += st.j_evals
        self.stats['iterations'] += st.iterations
        self.stats['minimizations'] += 1

    def run(self):
        cfg = self.cfg
        if self.face and self.optimize_betas and not self.face_with_free_shape:
            raise NotImplementedError('optimize_face with optimize_betas (chmosh.py:287-291): face_with_free_shape=True')
        extra_rigid = bool(cfg.opt_settings.get('extra_initial_rigid_adjustment', False))
        if extra_rigid and not self.reference_options:
            raise NotImplementedError('extra_initial_rigid_adjustment needs reference_options=True')
        self.rigid_adjust()
        if extra_rigid:
            self.extra_rigid_adjust()
        free_betas = self.optimize_betas
        ann = list(cfg.opt_settings.weights['stagei_wt_annealing'])
        errs = {}
        for tidx, a in enumerate(ann):
            detailed = tidx > len(ann) - 3                                                      # chmosh.py:311
            wts = self.weights_for(a)
            pose_ids = self.pose_ids_for(detailed)
            free_expr = detailed and self.face
            # (the keyword only where it is set: subclasses may override residual with the arguments before it)
            kw = {'free_expr': True} if free_expr else {}

            def obj(x, want_jac):
                return self.residual(x, want_jac, pose_ids, free_betas, wts, detailed, **kw)

            x, st = minimize_dogleg(obj, self.get_x(pose_ids, free_betas, free_expr), e_3=float(cfg.opt_settings.stagei_lr),
                                    delta_0=0.5, maxiter=int(cfg.opt_settings.maxiter))
            self.set_x(x, pose_ids, free_betas, free_expr)
            self._count(st)
            errs = {}
            self.residual(x, False, pose_ids, free_betas, wts, detailed, errs, **kw)
        return errs


def mosh_stagei(stagei_frames: List[Dict[str, np.ndarray]], cfg, betas_fname=None, v_template_fname=None, *, marker_meta=None,
                face_with_free_shape=False, reference_options=False, robust_data_sigma=None) -> dict:
    """Same inputs and return layout as the reference (chmosh.py:83-85,436-455), with the keywords of the product's
    ``mosh_stagei``; ``marker_meta`` is what ``marker_layout_load(cfg.dirs.marker_layout.fname, ...)`` returns
    (chmosh.py:121-125; layout tooling is out of scope).  With the face fitted the expressions of every picked frame are
    ``stagei_debug_details['opt_models_expression']``."""
    betas = np.load(betas_fname)['betas'] if betas_fname is not None else None
    v_template = None
    if v_template_fname is not None:
        from moshpp_b200.chmosh import _read_vertices       # host IO helper shared with the product
        v_template = _read_vertices(v_template_fname)
    s = StageISolver(stagei_frames, cfg, marker_meta, betas=betas, v_template=v_template, face_with_free_shape=face_with_free_shape,
                     reference_options=reference_options, robust_data_sigma=robust_data_sigma)
    errs = s.run()
    can_v = s.can_v()
    _, closest = NearestNeighbors(algorithm='kd_tree', n_neighbors=1).fit(can_v).kneighbors(s.ml)      # chmosh.py:422-424
    sims_all = s.markers_sim_all()
    dbg = {'opt_models_trans': [t.copy() for t in s.trans], 'opt_models_pose': [p.copy() for p in s.pose], 'stagei_errs': errs,
           'stagei_markers_sim_all': sims_all, 'stagei_markers_sim': [sims_all[f][s.lm_ids[f]] for f in range(s.n_frames)],
           'stagei_markers_obs': s.obs, 'stagei_labels_obs': s.labels_obs, 'oracle_stats': dict(s.stats)}
    if s.face:
        dbg['opt_models_expression'] = [e.copy() for e in s.expr]
    return {'betas': s.betas.copy(), 'markers_latent': s.ml.copy(), 'latent_labels': s.latent_labels, 'marker_meta': marker_meta,
            'markers_latent_vids': {l: int(c[0]) for l, c in zip(s.latent_labels, closest.tolist())}, 'stagei_debug_details': dbg}
