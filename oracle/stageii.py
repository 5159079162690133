"""Sequential Stage-II driver in float64 numpy (oracle; test infrastructure only).

Restates chmosh.py:458-741 -- the frame loop, the per-frame weights (596-609), the objective
dictionary (612-626, 681-699), the first-frame schedule (629-655), Step 1 (665-671), Step 2
(676-705) and the output packing (712-741) -- on top of lbs.py / markers.py / prior.py / rigid.py /
dogleg.py.  Known reference quirks that are kept on purpose: SURVEY.md Appendix B items 1, 2, 8, 9.

Modes
  ``lean``            evaluates only the <= 3M vertices the markers touch.
  ``reference_cost``  evaluates the full mesh and the dense 3V x P Jacobian on every evaluation and
                      then selects rows, i.e. the reference's cost structure (SURVEY.md 3.2); used
                      as the CPU baseline.  Both modes give the same numbers (tests/test_oracle_*).

``chunk=(L, W[, W_full])`` emulates the device's parallel-in-time schedule: frames are cut into chunks of L,
each solved like an independent sequence that starts W solved frames early, the last W_full of them with the
full per-frame schedule and the earlier ones with one Step-2 iteration (DESIGN.md "Chunked schedule").
``chunk=None`` is the reference's single sequential pass.

DMPL with SMPL-X is rejected by the reference (chmosh.py:508-509); BASELINE config 3 asks for it, so
``allow_smplx_dmpl=True`` lifts the assert and defines it by SURVEY.md Appendix A (extra beta
columns that also move the joints).  optimize_face is restated: the jaw joins Step 2 with its poseF term and the expression
coefficients are free with their expr term (chmosh.py:560-566,685-689).

Model types: the SMPL families, MANO, the horse and the dog (an LBS body without hands, its max-mixture prior over the pose
ids of chmosh.py:574-579).  ``robust_data_sigma``: the product's Geman-McClure data term (robust.py); None, the default, is
the reference's least-squares term.
"""
from __future__ import annotations

import pickle
import time
from typing import Dict, List, Optional, Tuple

import numpy as np

from .dogleg import minimize_dogleg
from .lbs import LBS, OracleModel
from .markers import TransformedCoeffs, transformed_lms
from .prior import DOG_POSE_IDS, HORSE_JANGLES_IDS, HORSE_JANGLES_SIGNS, create_body_prior, horse_joint_angles
from .rigid import perform_rigid_adjustment
from .robust import gm_dpsi, gm_psi

NUM_TRAIN_MARKERS = 46   # chmosh.py:460


class _Objective:
    """r(x), J(x) of one frame for the current free-variable set and term dictionary."""

    def __init__(self, solver, obs, vis_idx, terms, free_pose_ids, free_dmpl):
        self.s = solver
        self.obs = obs
        self.vis = vis_idx
        self.terms = terms                # ordered list of (name, payload)
        self.pose_ids = np.asarray(free_pose_ids, dtype=np.int64)
        self.free_dmpl = free_dmpl
        self.n = 3 + len(self.pose_ids) + (solver.nd if free_dmpl else 0)   # free_dmpl: the whole linear block (DMPL, expressions)

    def x0(self):
        s = self.s
        parts = [s.trans, s.pose[self.pose_ids]]
        if self.free_dmpl:
            parts.append(s.betas[s.lin_ids])
        return np.concatenate(parts)

    def assign(self, x):
        s = self.s
        s.trans = x[:3].copy()
        s.pose[self.pose_ids] = x[3:3 + len(self.pose_ids)]
        if self.free_dmpl:
            s.betas[s.lin_ids] = x[3 + len(self.pose_ids):]

    def __call__(self, x, want_jac):
        s = self.s
        self.assign(x)
        npi = len(self.pose_ids)
        ev = s.evaluate(want_jac)
        rs, Js = [], []
        for name, payload in self.terms:
            if name == 'data':
                wt = payload
                if s.robust_sigma is None:
                    r = ((ev['markers'][self.vis] - self.obs) * wt).reshape(-1)
                else:
                    e = (ev['markers'][self.vis] - self.obs).reshape(-1)
                    r = wt * gm_psi(e, s.robust_sigma)
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    dm_pose = ev['dm_pose'][self.vis].reshape(-1, s.model.pose_size)
                    J[:, :3] = np.tile(np.eye(3), (len(self.vis), 1)) * wt
                    J[:, 3:3 + npi] = dm_pose[:, self.pose_ids] * wt
                    if self.free_dmpl:
                        J[:, 3 + npi:] = ev['dm_beta'][self.vis].reshape(-1, s.nd) * wt
                    if s.robust_sigma is not None:
                        J *= gm_dpsi(e, s.robust_sigma)[:, None]
            elif name == 'poseB':
                wt = payload
                xb = s.pose[s.body_ids]
                r = s.prior.r(xb) * wt
                if want_jac:
                    Jp = s.prior.dr_wrt_x(xb) * wt
                    J = np.zeros((r.size, self.n))
                    col = {pid: c for c, pid in enumerate(self.pose_ids)}
                    for bi, pid in enumerate(s.body_ids):
                        if pid in col:
                            J[:, 3 + col[pid]] = Jp[:, bi]
            elif name == 'poseB_jangles':                                                          # chmosh.py:615-617
                wt = payload
                xb = s.pose[s.body_ids]
                r = horse_joint_angles(xb) * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    col = {pid: c for c, pid in enumerate(self.pose_ids)}
                    for ri, (bi, sg) in enumerate(zip(HORSE_JANGLES_IDS, HORSE_JANGLES_SIGNS)):
                        pid = s.body_ids[bi]
                        if pid in col:
                            J[ri, 3 + col[pid]] = 2.0 * sg * r[ri]
            elif name == 'velo':
                wt, target = payload
                r = (s.pose - target) * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    J[self.pose_ids, 3 + np.arange(npi)] = wt
            elif name == 'poseH':
                wt = payload
                r = s.pose[s.finger_ids] * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    col = {pid: c for c, pid in enumerate(self.pose_ids)}
                    for ri, pid in enumerate(s.finger_ids):
                        if pid in col:
                            J[ri, 3 + col[pid]] = wt
            elif name == 'extrap_dmpl':
                wt, target = payload
                r = (s.betas[s.dmpl_ids] - target) * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    if self.free_dmpl:
                        J[:, 3 + npi:3 + npi + s.n_dm] = np.eye(s.n_dm) * wt
            elif name == 'dmpl':
                wt = payload
                r = s.betas[s.dmpl_ids] * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    if self.free_dmpl:
                        J[:, 3 + npi:3 + npi + s.n_dm] = np.eye(s.n_dm) * wt
            elif name == 'poseF':                                                                  # chmosh.py:685-686
                wt = payload
                r = s.pose[s.face_ids] * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    col = {pid: c for c, pid in enumerate(self.pose_ids)}
                    for ri, pid in enumerate(s.face_ids):
                        if pid in col:
                            J[ri, 3 + col[pid]] = wt
            elif name == 'expr':                                                                   # chmosh.py:687
                wt = payload
                r = s.betas[s.expr_ids] * wt
                if want_jac:
                    J = np.zeros((r.size, self.n))
                    if self.free_dmpl:
                        J[:, 3 + npi + s.n_dm:] = np.eye(len(s.expr_ids)) * wt
            else:
                raise KeyError(name)
            rs.append(r)
            if want_jac:
                Js.append(J)
        r = np.concatenate(rs)
        if want_jac:
            return r, np.vstack(Js)
        return r

    def term_sse(self):
        ev = self.s.evaluate(False)
        out = {}
        for name, payload in self.terms:
            s = self.s
            if name == 'data':
                e = ev['markers'][self.vis] - self.obs
                if s.robust_sigma is not None:
                    e = gm_psi(e, s.robust_sigma)
                out[name] = float(((e * payload) ** 2).sum())
            elif name == 'poseB':
                out[name] = float(((s.prior.r(s.pose[s.body_ids]) * payload) ** 2).sum())
            elif name == 'poseB_jangles':
                out[name] = float(((horse_joint_angles(s.pose[s.body_ids]) * payload) ** 2).sum())
            elif name == 'velo':
                out[name] = float((((s.pose - payload[1]) * payload[0]) ** 2).sum())
            elif name == 'poseH':
                out[name] = float(((s.pose[s.finger_ids] * payload) ** 2).sum())
            elif name == 'extrap_dmpl':
                out[name] = float((((s.betas[s.dmpl_ids] - payload[1]) * payload[0]) ** 2).sum())
            elif name == 'dmpl':
                out[name] = float(((s.betas[s.dmpl_ids] * payload) ** 2).sum())
            elif name == 'poseF':
                out[name] = float(((s.pose[s.face_ids] * payload) ** 2).sum())
            elif name == 'expr':
                out[name] = float(((s.betas[s.expr_ids] * payload) ** 2).sum())
        return out


class StageIISolver:
    """State of ``opt_model`` + everything chmosh.py:488-579 sets up before the frame loop."""

    def __init__(self, cfg, markers_latent, latent_labels, betas, marker_meta, mode='lean',
                 allow_smplx_dmpl=True, robust_data_sigma=None):
        sm, mp = cfg.surface_model, cfg.moshpp
        self.cfg = cfg
        self.mode = mode
        self.robust_sigma = robust_data_sigma          # None: the reference's least-squares data term
        self.latent_labels = list(latent_labels)
        self.optimize_fingers = bool(mp.optimize_fingers)
        self.optimize_face = bool(mp.optimize_face)
        # chmosh.py:475-486: gate finger / face optimisation on the layout / available labels
        if self.optimize_face:
            if not np.any(['face' in m for m in marker_meta['marker_type_mask'].keys()]):
                self.optimize_face = False
            elif not np.any([('face' in t) and l in self.latent_labels for l, t in marker_meta['marker_type'].items()]):
                self.optimize_face = False
        if self.optimize_fingers:
            if not np.any(['finger' in m for m in marker_meta['marker_type_mask'].keys()]):
                self.optimize_fingers = False
            elif not np.any([('finger' in t) and l in self.latent_labels for l, t in marker_meta['marker_type'].items()]):
                self.optimize_fingers = False
        self.model = OracleModel(sm.fname, pose_hand_prior_fname=mp.pose_hand_prior_fname,
                                 use_hands_mean=sm.use_hands_mean, dof_per_hand=sm.dof_per_hand,
                                 surface_model_type=sm.type)
        m = self.model
        assert m.model_type == sm.type
        self.prior = create_body_prior(m.model_type, mp.pose_body_prior_fname)
        self.betas = np.zeros(m.n_betas_model)
        self.betas[:sm.num_betas] = np.asarray(betas)[:sm.num_betas]                            # chmosh.py:499-500
        self.pose = np.zeros(m.pose_size)
        self.trans = np.zeros(3)

        can = LBS(m, None)(np.zeros(m.pose_size), self.betas, np.zeros(3))                      # can_model.r
        self.tc = TransformedCoeffs(can, markers_latent)                                        # chmosh.py:502
        self.n_markers = len(markers_latent)

        self.nd = 0
        self.dmpl_ids = np.zeros(0, dtype=np.int64)
        self.optimize_dynamics = bool(mp.optimize_dynamics)
        if self.optimize_dynamics:                                                              # chmosh.py:507-514
            if not allow_smplx_dmpl:
                assert sm.type in ['smpl', 'smplh'], NotImplementedError('DMPLs are currently only supported by smpl and smplh models')
            total = sm.num_betas + sm.num_dmpls
            with open(sm.dmpl_fname, 'rb') as f:
                dmpl_pcs = pickle.load(f)['eigvec']
            m.shapedirs[:, :, sm.num_betas:total] = dmpl_pcs[:, :, :sm.num_dmpls]
            self.nd = int(sm.num_dmpls)
            self.dmpl_ids = np.arange(sm.num_betas, total)
        self.n_dm = self.nd
        # expression coefficients (chmosh.py:560-566): betas[exp_start : exp_start + num_expressions], free in Step 2
        self.expr_ids = np.zeros(0, dtype=np.int64)
        self.exp_start = 0
        if self.optimize_face and sm.type == 'smplx':
            self.exp_start = int(sm.betas_expr_start_id)
            self.expr_ids = np.arange(self.exp_start, self.exp_start + int(sm.num_expressions))
            assert self.expr_ids[-1] < m.n_betas_model, 'the model has no such expression components'
        self.lin_ids = np.concatenate([self.dmpl_ids, self.expr_ids]).astype(np.int64)
        self.nd = len(self.lin_ids)

        if mode == 'lean':
            self.vids = self.tc.vids
            self.lbs = LBS(m, self.vids)
            lut = {v: i for i, v in enumerate(self.vids)}
            self.tri = np.vectorize(lut.get)(self.tc.closest[:, :3])
        elif mode == 'reference_cost':
            self.lbs = LBS(m, None)
            self.tri = self.tc.closest[:, :3]
        else:
            raise ValueError(mode)

        # pose-id partitions, chmosh.py:548-571
        all_ids = list(range(m.pose_size))
        self.root_ids = all_ids[:3]
        self.body_ids: List[int] = []
        self.finger_ids: List[int] = []
        self.face_ids: List[int] = []
        if sm.type == 'smpl':
            self.body_ids = all_ids[3:]
        elif sm.type == 'smplh':
            self.body_ids = all_ids[3:66]
            if self.optimize_fingers:
                self.finger_ids = all_ids[66:]
        elif sm.type == 'smplx':
            self.body_ids = all_ids[3:66]
            if self.optimize_face:
                self.face_ids = all_ids[66:69]                                                   # jaw only (line 564)
            if self.optimize_fingers:
                self.finger_ids = all_ids[75:]
        elif sm.type == 'mano':
            self.finger_ids = all_ids[3:]
        elif sm.type == 'animal_horse':
            self.body_ids = all_ids[3:84]                                                       # line 572-573
        elif sm.type == 'animal_dog':
            self.body_ids = [all_ids[i] for i in DOG_POSE_IDS]                                  # lines 574-579
        else:
            raise NotImplementedError(sm.type)
        ids = self.root_ids + self.body_ids
        if len(self.body_ids) and not mp.optimize_toes:
            ids = list(set(ids).difference(set(all_ids[30:36])))                                # lines 645-647
        self.step1_ids = sorted(ids)
        ids2 = list(ids)
        if self.optimize_fingers:
            ids2 += self.finger_ids
        if self.optimize_face:
            ids2 += self.face_ids                                                                # line 689
        self.step2_ids = sorted(set(ids2))                                                      # line 691
        self.wts = cfg.opt_settings.weights
        self.maxiter = int(cfg.opt_settings.maxiter)
        self.stats = dict(r_evals=0, j_evals=0, iterations=0, minimizations=0)

    # ---- one evaluation of opt_model.r / markers_sim (and Jacobians)
    def evaluate(self, want_jac):
        res = self.lbs(self.pose, self.betas, self.trans, want_jac, beta_ids=self.lin_ids)
        verts = res[0] if want_jac else res
        t = self.tri
        if not want_jac:
            return {'markers': transformed_lms(self.tc, verts[t[:, 0]], verts[t[:, 1]], verts[t[:, 2]])}
        _, dv_pose, dv_beta = res
        mk, loc = transformed_lms(self.tc, verts[t[:, 0]], verts[t[:, 1]], verts[t[:, 2]], True)
        dm_pose = np.zeros((self.n_markers, 3, self.model.pose_size))
        dm_beta = np.zeros((self.n_markers, 3, self.nd))
        for k in range(3):
            L = loc[:, :, 3 * k:3 * k + 3]
            dm_pose += np.einsum('mcd,mdp->mcp', L, dv_pose[t[:, k]])
            if self.nd:
                dm_beta += np.einsum('mcd,mdb->mcb', L, dv_beta[t[:, k]])
        return {'markers': mk, 'dm_pose': dm_pose, 'dm_beta': dm_beta}

    def _minimize(self, objective, e_3, maxiter=None):
        x, st = minimize_dogleg(objective, objective.x0(), e_3=e_3, delta_0=0.5, maxiter=maxiter or self.maxiter)
        objective.assign(x)
        self.stats['r_evals'] += st.r_evals
        self.stats['j_evals'] += st.j_evals
        self.stats['iterations'] += st.iterations
        self.stats['minimizations'] += 1
        return st

    def reset(self):
        self.pose[:] = 0.0
        self.trans[:] = 0.0
        if self.nd:
            self.betas[self.lin_ids] = 0.0

    def frame_terms(self, n_visible: int, velo_target=None, dmpl_target=None):
        """The objective of one frame (chmosh.py:596-626, 681-699) as a list of [name, payload] terms: the Step-2 list, of
        which Step 1 minimises the first ``n_step1``.  ``n_visible`` (markers seen in the frame) sets the weights;
        ``velo_target`` (2 pose[t-1] - pose[t-2]) and ``dmpl_target`` switch the velocity and DMPL-extrapolation terms
        on.  Returns (terms, n_step1)."""
        w = self.wts
        M = self.n_markers
        n_missing = float(M - n_visible)
        anneal = 1.0
        if n_missing > 0:
            anneal = anneal + (n_missing / M) * w['stageii_wt_annealing']
        wt_data = w['stageii_wt_data'] * (NUM_TRAIN_MARKERS / n_visible)
        wt_pose = w['stageii_wt_poseB'] * anneal

        terms = [['data', wt_data]]
        if len(self.body_ids):
            terms.append(['poseB', wt_pose])
            if self.model.model_type == 'animal_horse':
                terms.append(['poseB_jangles', wt_pose * 2.])                                    # lines 615-617
        if velo_target is not None:
            terms.append(['velo', (w['stageii_wt_velo'], velo_target)])                          # line 626
        n_step1 = len(terms)
        if self.optimize_fingers:
            terms.append(['poseH', w['stageii_wt_poseH'] * anneal])
        if self.optimize_face and len(self.face_ids):
            terms.append(['poseF', w['stageii_wt_poseF'] * anneal])
            terms.append(['expr', w['stageii_wt_expr']])
        if self.optimize_dynamics:
            if dmpl_target is not None:
                terms.append(['extrap_dmpl', (6.0, dmpl_target)])                                # line 697 (App. B-1)
            terms.append(['dmpl', w['stageii_wt_dmpl']])
        return terms, n_step1

    def solve_range(self, obs_frames: List[Optional[Tuple[np.ndarray, np.ndarray]]], emit_from: int = 0,
                    light_until: int = 0, on_frame=None):
        """The frame loop chmosh.py:584-724 over ``obs_frames`` (each ``(vis_idx, obs m x 3)`` or None for a
        frame without visible markers).  Frames before ``emit_from`` are solved but not reported.  Device-schedule
        emulation only (not reference behaviour): frames before ``light_until`` other than the first solved one are
        tracked with a single dog-leg iteration of the Step-2 problem (DESIGN.md section 4)."""
        pose_prev = None
        first = True
        out = []
        for fi, fr in enumerate(obs_frames):
            if fr is None:                                                                       # lines 586-588
                continue
            vis, obs = fr
            velo_target = None if pose_prev is None else self.pose + (self.pose - pose_prev)     # line 626
            dmpl_target = None
            if not first:
                pose_prev = self.pose.copy()                                                     # lines 656-659
                if self.optimize_dynamics:
                    # line 697 (App. B-1); Step 1 leaves the coefficients where they are, so the target is known here
                    dmpl_prev = self.betas[self.dmpl_ids].copy()
                    cur = self.betas[self.dmpl_ids]
                    dmpl_target = cur + (cur - dmpl_prev)
            terms, n_step1 = self.frame_terms(len(vis), velo_target, dmpl_target)
            step1 = terms[:n_step1]                     # (the same [name, payload] lists: Step 1 sees the schedule below)

            was_first = first
            if first:
                sim = self.evaluate(False)['markers'][vis]
                rv, T = perform_rigid_adjustment(sim, obs)                                       # line 634
                self.pose[:3] = rv
                self.trans[:] = T
                wt_pose = terms[1][1] if len(self.body_ids) else None
                for scale in (10., 5., 1.):
                    if len(self.body_ids):
                        wt_first = scale * wt_pose
                        terms[1][1] = wt_first
                        if self.model.model_type == 'animal_horse':
                            terms[2][1] = wt_first * 2.                                          # lines 640-643
                    self._minimize(_Objective(self, obs, vis, step1, self.step1_ids, False), 1e-3)
                first = False

            light = (not was_first) and fi < light_until
            if not light:
                self._minimize(_Objective(self, obs, vis, step1, self.step1_ids, False), 1e-2)    # Step 1

            obj2 = _Objective(self, obs, vis, terms, self.step2_ids, self.nd > 0)
            self._minimize(obj2, 1e-2, maxiter=1 if light else None)                             # Step 2

            if on_frame is not None:
                on_frame(fi)                  # bench.py: wall-clock stamp after every solved frame
            if fi >= emit_from:
                errs = obj2.term_sse()
                mk = self.evaluate(False)['markers'][vis]
                out.append(dict(fidx=fi, errs=errs, markers_sim=mk.copy(), markers_obs=obs.copy(), vis=vis,
                                fullpose=self.model.fullpose(self.pose), pose=self.pose.copy(),
                                trans=self.trans.copy(),
                                dmpls=self.betas[self.dmpl_ids].copy() if self.optimize_dynamics else None,
                                expression=self.betas[self.exp_start:].copy() if len(self.expr_ids) else None))   # line 724: the whole tail
        return out


def frames_from_mocap(markers, labels, latent_labels):
    """``markers_asdict`` + the per-frame stacking of chmosh.py:582-594 on dense arrays.
    markers: F x L x 3 in metres with missing samples already zeroed (mocap_interface.py:223-225)."""
    cols = {}
    for i, l in enumerate(labels):
        cols.setdefault(l, []).append(i)
    avail = np.logical_and(np.isnan(markers).sum(-1) == 0, (markers == 0).sum(-1) != 3)   # mocap_interface.py:277
    frames = []
    for t in range(markers.shape[0]):
        # markers_asdict writes the frame's dictionary in column order and only for available samples
        # (mocap_interface.py:262-271): of several columns with one label the last AVAILABLE one wins
        pick = {}
        for li, l in enumerate(latent_labels):
            for c in cols.get(l, ()):
                if avail[t, c]:
                    pick[li] = c
        vis = sorted(pick)
        if not vis:
            frames.append(None)
            continue
        obs = np.vstack([markers[t, pick[li]] for li in vis])
        frames.append((np.asarray(vis, dtype=np.int64), obs))
    return frames


def mosh_stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None,
                 *, mode='lean', chunk=None, max_frames=None, allow_smplx_dmpl=True, mocap=None, on_frame=None,
                 robust_data_sigma=None) -> dict:
    """Same signature and return layout as the reference (chmosh.py:458-459, 726-741).  ``robust_data_sigma`` (metres; the
    product's keyword): the data rows Geman-McClure robustified (robust.py) instead of least squares."""
    if mocap is None:
        # host IO adapter (outside the oracle's scope, SURVEY.md 8(f-1)); shared with the product
        from moshpp_b200.mocap_interface import MocapSession
        mocap = MocapSession(mocap_fname, mocap_unit=cfg.mocap.unit, mocap_rotate=cfg.mocap.rotate,
                             only_subjects=[cfg.mocap.subject_name] if cfg.mocap.multi_subject else None)
    solver = StageIISolver(cfg, markers_latent, latent_labels, betas, marker_meta, mode=mode,
                           allow_smplx_dmpl=allow_smplx_dmpl, robust_data_sigma=robust_data_sigma)
    n = len(mocap.markers)
    sel = list(range(cfg.mocap.start_fidx, n if cfg.mocap.end_fidx == -1 else cfg.mocap.end_fidx, cfg.mocap.ds_rate))
    if max_frames is not None:
        sel = sel[:max_frames]
    frames = frames_from_mocap(mocap.markers[sel], mocap.labels, solver.latent_labels)
    t0 = time.time()
    if chunk is None:
        per = solver.solve_range(frames, on_frame=on_frame)
    else:
        L, W = chunk[:2]
        W_full = chunk[2] if len(chunk) > 2 and 0 <= chunk[2] <= W else W
        E = chunk[3] if len(chunk) > 3 and L < len(frames) else 0      # mosh2_schedule.first_extra: the first chunk is longer
        per = []
        starts = [0] + list(range(L + E, len(frames), L)) if E > 0 else list(range(0, len(frames), L))
        for ci, s in enumerate(starts):
            s_end = starts[ci + 1] if ci + 1 < len(starts) else len(frames)
            # the warm-up is counted in solved frames (frames with a visible marker), walking back from the chunk
            lo, full_from, cnt = s, s, 0
            while lo > 0 and cnt < W:
                lo -= 1
                if frames[lo] is not None:
                    cnt += 1
                    if cnt <= W_full:
                        full_from = lo
            while lo < s and frames[lo] is None:
                lo += 1
            if cnt < W:
                full_from = lo      # the walk-back reached the first frame: the chunk is the sequential recursion itself
            solver.reset()
            res = solver.solve_range(frames[lo:s_end], emit_from=s - lo, light_until=full_from - lo)
            for r in res:
                r['fidx'] += lo
            per += res
    elapsed = time.time() - t0

    errs: Dict[str, list] = {}
    for r in per:
        for k, v in r['errs'].items():
            errs.setdefault(k, []).append(v)
    dbg = {
        'stageii_errs': {k: np.array(v) for k, v in errs.items()},
        'markers_sim': [r['markers_sim'] for r in per],
        'markers_obs': [r['markers_obs'] for r in per],
        'labels_obs': [[solver.latent_labels[i] for i in r['vis']] for r in per],
        'markers_orig': mocap.markers[sel],
        'labels_orig': mocap.labels,
        'mocap_fname': mocap_fname,
        'mocap_frame_rate': mocap.frame_rate,
        'mocap_time_length': mocap.time_length(),
        'oracle_stats': dict(solver.stats, elapsed=elapsed, frames=len(per)),
        'frame_ids': np.array([r['fidx'] for r in per]),
    }
    data = {'fullpose': np.array([r['fullpose'] for r in per]), 'trans': np.array([r['trans'] for r in per])}
    if solver.optimize_dynamics:
        data['dmpls'] = np.array([r['dmpls'] for r in per])
    if len(solver.expr_ids):                                                                    # chmosh.py:723-724,736
        data['expression'] = np.array([r['expression'] for r in per])
    data['stageii_debug_details'] = dbg
    data['_pose_reduced'] = np.array([r['pose'] for r in per])
    return data
