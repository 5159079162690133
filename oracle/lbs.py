"""SMPL-family forward + analytic Jacobians in float64 numpy (oracle; test infrastructure only).

Restates, for the Stage-II path:
  * ``load_surface_model`` / ``SmplModelLBS.__init__`` -- models/smpl_fast_derivatives.py:52-166,169-241
    (model-type rules, hand PCA ``selected_components``, ``hands_mean`` incl. MANO's inverted flag,
    v_shaped, J = J_regressor . v_shaped per axis).
  * ``verts_decorated`` (psbody.smpl, external; bs_type 'lrotmin', bs_style 'lbs') -- call site
    smpl_fast_derivatives.py:206-218 -- from the public SMPL formulation (SURVEY.md Appendix A.3).
  * ``lbs_derivatives_wrt_pose`` / ``_wrt_shape`` (external C++) and the PCA chain rule --
    smpl_fast_derivatives.py:246-263.

``LBS(model, rows=None)`` evaluates all V vertices (the reference's cost structure: full mesh and a
dense 3V x P Jacobian every evaluation); ``LBS(model, rows=vids)`` evaluates only the listed
vertices (the "lean" oracle).  Both run the same code, so row selection commutes by construction.
"""
from __future__ import annotations

import pickle
from typing import Optional, Sequence

import numpy as np

from .rigid import rodrigues

MODEL_TYPES = {69: 'smpl', 153: 'smplh', 162: 'smplx', 45: 'mano'}


class OracleModel:
    """Arrays of one body model + the pose parametrisation (smpl_fast_derivatives.py:52-145)."""

    def __init__(self, surface_model_fname, pose_hand_prior_fname=None, use_hands_mean=False,
                 dof_per_hand=12, v_template=None, surface_model_type=None):
        assert surface_model_fname.endswith('.pkl'), ValueError('surface_model_fname could only be a pkl file.')
        with open(surface_model_fname, 'rb') as f:
            dd = pickle.load(f, encoding='latin-1')
        njoint_parms = dd['posedirs'].shape[2] // 3
        self.model_type = surface_model_type or MODEL_TYPES[njoint_parms]
        assert dd['bs_style'] == 'lbs'
        if v_template is not None:
            dd['v_template'] = v_template
        if self.model_type in ('smplx', 'smplh'):
            self.body_dof = njoint_parms - 90 + 3
            assert pose_hand_prior_fname is not None and pose_hand_prior_fname.endswith('.npz')
            mp = np.load(pose_hand_prior_fname)
            cl, cr = mp['componentsl'], mp['componentsr']
            ml = mp['hands_meanl'] if use_hands_mean else np.zeros(cl.shape[1])
            mr = mp['hands_meanr'] if use_hands_mean else np.zeros(cr.shape[1])
            self.selected_components = np.vstack(
                (np.hstack((cl[:dof_per_hand], np.zeros_like(cl[:dof_per_hand]))),
                 np.hstack((np.zeros_like(cr[:dof_per_hand]), cr[:dof_per_hand]))))
            self.hands_mean = np.concatenate((ml, mr))
        elif self.model_type == 'mano':
            self.body_dof = 3
            hc = dd['hands_components']
            self.hands_mean = np.zeros(hc.shape[1]) if use_hands_mean else dd['hands_mean']   # sic (line 114)
            self.selected_components = np.vstack((hc[:dof_per_hand]))
        else:                           # smpl and the animal models (animal_horse, animal_dog): an LBS body without hands
            self.body_dof = njoint_parms + 3
            self.selected_components = np.zeros((0, 0))
            self.hands_mean = np.zeros(0)
        jreg = dd['J_regressor']
        self.J_regressor = np.asarray(jreg.toarray() if hasattr(jreg, 'toarray') else jreg, dtype=np.float64)
        self.v_template = np.asarray(dd['v_template'], dtype=np.float64)
        self.shapedirs = np.array(dd['shapedirs'], dtype=np.float64)       # copy: DMPL columns are overwritten
        self.posedirs = np.asarray(dd['posedirs'], dtype=np.float64)
        self.weights = np.asarray(dd['weights'], dtype=np.float64)
        kt = np.asarray(dd['kintree_table'])
        self.parents = kt[0].astype(np.int64)
        self.parents[0] = -1
        self.n_joints = kt.shape[1]
        self.n_betas_model = self.shapedirs.shape[-1]
        self.pose_size = self.body_dof + self.selected_components.shape[0]
        nj = self.n_joints
        self.subtree = np.eye(nj, dtype=bool)       # subtree[a, j] <=> j is a or a descendant of a
        for j in range(1, nj):
            a = self.parents[j]
            while a >= 0:
                self.subtree[a, j] = True
                a = self.parents[a]

    def fullpose(self, pose):
        """smpl_fast_derivatives.py:194-204."""
        pose = np.asarray(pose, dtype=np.float64)
        if self.selected_components.shape[0] == 0:
            return pose.copy()
        hand = pose[self.body_dof:].dot(self.selected_components)
        return np.concatenate((pose[:self.body_dof], self.hands_mean + hand))

    def dfullpose_dpose(self):
        """blockdiag(I, C^T): smpl_fast_derivatives.py:250-254."""
        pf, pr = 3 * self.n_joints, self.pose_size
        m = np.zeros((pf, pr))
        m[:self.body_dof, :self.body_dof] = np.eye(self.body_dof)
        if self.selected_components.shape[0]:
            m[self.body_dof:, self.body_dof:] = self.selected_components.T
        return m


class LBS:
    """verts(pose, betas, trans) and its Jacobians for all vertices or a row subset."""

    def __init__(self, model: OracleModel, rows: Optional[Sequence[int]] = None):
        self.m = model
        self.rows = None if rows is None else np.asarray(rows, dtype=np.int64)
        sel = slice(None) if rows is None else self.rows
        self.v_template = model.v_template[sel]
        self.shapedirs = model.shapedirs[sel]
        self.posedirs = model.posedirs[sel]
        self.weights = model.weights[sel]
        if rows is not None:
            # J = Jreg . (T + S beta) is linear in beta: fold the regressor once (algebraically
            # identical to smpl_fast_derivatives.py:186-191; the full-mesh mode below keeps the
            # reference's per-evaluation regression).
            self.J_t = model.J_regressor.dot(model.v_template)
            self.J_dirs = np.einsum('jv,vcb->jcb', model.J_regressor, model.shapedirs)

    def refresh_shapedirs(self):
        sel = slice(None) if self.rows is None else self.rows
        self.shapedirs = self.m.shapedirs[sel]
        if self.rows is not None:
            self.J_dirs = np.einsum('jv,vcb->jcb', self.m.J_regressor, self.m.shapedirs)

    def __call__(self, pose, betas, trans, want_jac=False, beta_ids=()):
        """Returns verts (S x 3) and, if want_jac, (dv/dpose S x 3 x P_red, dv/dbetas[beta_ids] S x 3 x nb)."""
        m = self.m
        nj = m.n_joints
        betas = np.asarray(betas, dtype=np.float64)
        nb = len(betas)
        v_shaped = self.v_template + self.shapedirs[:, :, :nb].dot(betas)
        if self.rows is None:
            J = m.J_regressor.dot(v_shaped)                       # per-axis MatVecMult, lines 187-191
            J_dirs = None
        else:
            J = self.J_t + self.J_dirs[:, :, :nb].dot(betas)
            J_dirs = self.J_dirs
        full = m.fullpose(pose)

        R = np.zeros((nj, 3, 3))
        dR = np.zeros((nj, 3, 3, 3))
        for j in range(nj):
            if want_jac:
                R[j], dR[j] = rodrigues(full[3 * j:3 * j + 3], True)
            else:
                R[j] = rodrigues(full[3 * j:3 * j + 3])
        posefeat = (R[1:] - np.eye(3)).reshape(-1)                 # lrotmin: vec_rowmajor(R_j - I), j >= 1
        v_posed = v_shaped + self.posedirs.dot(posefeat)

        Rg = np.zeros((nj, 3, 3))
        tg = np.zeros((nj, 3))
        Rg[0], tg[0] = R[0], J[0]
        for j in range(1, nj):
            a = m.parents[j]
            Rg[j] = Rg[a].dot(R[j])
            tg[j] = tg[a] + Rg[a].dot(J[j] - J[a])
        # p[v, j] = A_j [v_posed; 1],  A_j = G_j [I | -J_j]
        p = np.einsum('jcd,vjd->vjc', Rg, v_posed[:, None, :] - J[None, :, :]) + tg[None]
        W = self.weights
        verts = np.einsum('vj,vjc->vc', W, p) + np.asarray(trans, dtype=np.float64)[None]
        if not want_jac:
            return verts

        S = verts.shape[0]
        pf = 3 * nj
        # ---- rigid part: d/dw_{a,k} = u_{a,k} x sum_{j in subtree(a)} w_vj (p_vj - t_a)
        Wp = W[:, :, None] * p
        sub = m.subtree.astype(np.float64)
        q = np.einsum('aj,vjc->vac', sub, Wp) - (W.dot(sub.T))[:, :, None] * tg[None]
        dv_full = np.zeros((S, 3, pf))
        for a in range(nj):
            Rpar = np.eye(3) if a == 0 else Rg[m.parents[a]]
            for k in range(3):
                Om = dR[a, k].dot(R[a].T)                       # skew
                u = Rpar.dot(np.array([Om[2, 1], Om[0, 2], Om[1, 0]]))
                dv_full[:, :, 3 * a + k] = np.cross(u[None], q[:, a])
        # ---- pose-blend part: T_v^lin . posedirs . d posefeat / dw
        Rskin = np.einsum('vj,jcd->vcd', W, Rg)
        Pd = self.posedirs.reshape(S, 3, nj - 1, 9)
        E = np.einsum('vdjn,jkn->vdjk', Pd, dR[1:].reshape(nj - 1, 3, 9))
        dv_full[:, :, 3:] += np.einsum('vcd,vdjk->vcjk', Rskin, E).reshape(S, 3, pf - 3)
        dv_pose = dv_full.dot(m.dfullpose_dpose())               # the np.matmul at smpl_fast_derivatives.py:255

        dv_beta = np.zeros((S, 3, len(beta_ids)))
        if len(beta_ids):
            bi = np.asarray(beta_ids)
            Sb = self.shapedirs[:, :, bi]                        # d v_shaped / d beta
            if J_dirs is None:
                Jb = np.einsum('jv,vcb->jcb', m.J_regressor, self.shapedirs[:, :, bi])
            else:
                Jb = J_dirs[:, :, bi]
            dtg = np.zeros((nj, 3, len(bi)))
            dtg[0] = Jb[0]
            for j in range(1, nj):
                a = m.parents[j]
                dtg[j] = dtg[a] + Rg[a].dot(Jb[j] - Jb[a])
            dp = np.einsum('jcd,vjdb->vjcb', Rg, Sb[:, None] - Jb[None]) + dtg[None]
            dv_beta = np.einsum('vj,vjcb->vcb', W, dp)
        return verts, dv_pose, dv_beta
