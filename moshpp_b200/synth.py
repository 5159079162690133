"""Procedural fixtures: body models, priors, marker layouts, motions and mocap files.

No body-model, prior, DMPL or mocap file exists in the build environment (SURVEY.md 8(c)) and
none may be copied from the reference, so tests and ``bench.py`` run on seeded procedural data in
the reference's own on-disk formats (SURVEY.md Appendix C):

* model pickle: ``v_template, shapedirs, posedirs, weights, J_regressor, kintree_table, f,
  bs_style='lbs', bs_type='lrotmin'`` (+ ``hands_components, hands_mean`` for MANO),
* hand prior npz ``componentsl/r, hands_meanl/r``; body prior pkl ``covars, means, weights``;
  DMPL pkl ``eigvec``.

The geometry is a capsule humanoid over the public SMPL / SMPL-H / SMPL-X / MANO kinematic trees
(24 / 52 / 55 / 16 joints) with exactly 6890 / 6890 / 10475 / 778 vertices (SMPL-X keeps the
1092-vertex eyeball tail block the marker attachment must skip).  Seeds follow SURVEY.md 8(d).

This module generates data only; it holds a small vectorised LBS forward to synthesise
observations, checked against the oracle in tests/test_synth.py.
"""
from __future__ import annotations

import hashlib
import os
import pickle
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp

from . import pack as _pack

SEED_MODEL, SEED_LAYOUT, SEED_MOTION, SEED_NOISE, SEED_DROPOUT = 1234, 2345, 3456, 4567, 5678

STD46 = ('ARIEL C7 CLAV LANK LBAK LBHD LBSH LBWT LELB LFHD LFRM LFSH LFWT LHEE LIWR LKNE LMT1 LMT5 LOWR LSHN '
         'LTHI LTOE LUPA RANK RBAK RBHD RBSH RBWT RELB RFHD RFRM RFSH RFWT RHEE RIWR RKNE RMT1 RMT5 ROWR RSHN '
         'RTHI RTOE RUPA STRN T10 T8').split()
FINGER6 = ['IDX1', 'IDX3', 'MID3', 'RNG3', 'PNK3', 'THM3']
FINGER10 = ['IDX1', 'IDX2', 'IDX3', 'MID1', 'MID2', 'MID3', 'RNG3', 'PNK3', 'THM2', 'THM3']

# --------------------------------------------------------------------------------------
# skeletons (public kinematic trees; rest pose is a rough T-pose, metres, y up, x to the left)
# --------------------------------------------------------------------------------------
_BODY22 = np.array([
    [0.00, -0.22, 0.02], [0.07, -0.31, 0.01], [-0.07, -0.31, 0.01], [0.00, -0.11, -0.01],
    [0.10, -0.69, 0.02], [-0.10, -0.69, 0.02], [0.00, 0.02, 0.02], [0.09, -1.09, -0.02],
    [-0.09, -1.09, -0.02], [0.00, 0.07, 0.03], [0.11, -1.15, 0.10], [-0.11, -1.15, 0.10],
    [0.00, 0.28, 0.00], [0.08, 0.19, 0.00], [-0.08, 0.19, 0.00], [0.00, 0.35, 0.04],
    [0.17, 0.23, -0.01], [-0.17, 0.23, -0.01], [0.43, 0.22, -0.03], [-0.43, 0.22, -0.03],
    [0.68, 0.23, -0.03], [-0.68, 0.23, -0.03]])
_BODY22_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19]
_BODY22_RADII = [0.13, 0.075, 0.075, 0.125, 0.05, 0.05, 0.12, 0.04, 0.04, 0.12, 0.035, 0.035,
                 0.05, 0.06, 0.06, 0.09, 0.045, 0.045, 0.035, 0.035, 0.028, 0.028]


def _hand_joints(wrist: np.ndarray, side: float):
    """15 finger joints (index, middle, pinky, ring, thumb; 3 each) for a hand pointing along side*x."""
    pos, par = [], []
    fingers = [(+0.025, 0.092), (+0.005, 0.095), (-0.035, 0.082), (-0.015, 0.090)]
    seg = [0.035, 0.025, 0.020]
    for z, x0 in fingers:
        base = wrist + np.array([side * x0, 0.0, z])
        p = base.copy()
        for k in range(3):
            pos.append(p.copy())
            par.append(-1 if k == 0 else len(pos) - 2)
            p = p + np.array([side * seg[k], 0.0, 0.0])
    d = np.array([side * 0.6, -0.2, 0.77])
    d /= np.linalg.norm(d)
    p = wrist + np.array([side * 0.03, -0.01, 0.035])
    for k, L in enumerate([0.035, 0.03, 0.025]):
        pos.append(p.copy())
        par.append(-1 if k == 0 else len(pos) - 2)
        p = p + d * L
    return np.array(pos), par


def skeleton(model_type: str):
    """Returns (joint positions nJ x 3, parents, capsule radius per joint)."""
    if model_type == 'smpl':
        pos = np.vstack([_BODY22, [[0.77, 0.22, -0.04], [-0.77, 0.22, -0.04]]])
        par = _BODY22_PARENTS + [20, 21]
        rad = _BODY22_RADII + [0.025, 0.025]
        return pos, np.array(par), np.array(rad)
    if model_type in ('smplh', 'smplx'):
        pos = [_BODY22]
        par = list(_BODY22_PARENTS)
        rad = list(_BODY22_RADII)
        if model_type == 'smplx':
            pos.append(np.array([[0.0, 0.33, 0.06], [0.032, 0.40, 0.10], [-0.032, 0.40, 0.10]]))
            par += [15, 15, 15]
            rad += [0.03, 0.012, 0.012]
        for wrist_id, side in ((20, 1.0), (21, -1.0)):
            hp, hpar = _hand_joints(_BODY22[wrist_id], side)
            base = len(par)
            pos.append(hp)
            par += [wrist_id if p < 0 else base + p for p in hpar]
            rad += [0.009] * 15
        return np.vstack(pos), np.array(par), np.array(rad)
    if model_type == 'mano':
        wrist = np.zeros(3)
        hp, hpar = _hand_joints(wrist, 1.0)
        pos = np.vstack([wrist[None], hp])
        par = [-1] + [0 if p < 0 else 1 + p for p in hpar]
        rad = [0.03] + [0.009] * 15
        return pos, np.array(par), np.array(rad)
    if model_type == 'animal_horse':
        return _HORSE35, np.array(_HORSE35_PARENTS), np.array(_HORSE35_RADII)
    raise ValueError(model_type)


# a quadruped with 35 joints: 28 body joints (pose ids 0..83 are optimised), then tail (3), mouth, ears (2), forelock
_HORSE35 = np.array([
    [-0.50, 1.10, 0.0], [-0.25, 1.15, 0.0], [0.00, 1.15, 0.0], [0.25, 1.15, 0.0], [0.50, 1.15, 0.0],
    [0.70, 1.35, 0.0], [0.85, 1.55, 0.0], [1.00, 1.65, 0.0],
    [0.50, 0.95, 0.15], [0.50, 0.65, 0.15], [0.50, 0.35, 0.15], [0.50, 0.10, 0.15],
    [0.50, 0.95, -0.15], [0.50, 0.65, -0.15], [0.50, 0.35, -0.15], [0.50, 0.10, -0.15],
    [-0.50, 0.90, 0.15], [-0.50, 0.60, 0.15], [-0.55, 0.30, 0.15], [-0.50, 0.08, 0.15],
    [-0.50, 0.90, -0.15], [-0.50, 0.60, -0.15], [-0.55, 0.30, -0.15], [-0.50, 0.08, -0.15],
    [0.10, 1.00, 0.0], [-0.20, 1.00, 0.0], [0.62, 1.25, 0.0], [-0.62, 1.20, 0.0],
    [-0.65, 1.10, 0.0], [-0.80, 1.00, 0.0], [-0.90, 0.85, 0.0], [1.12, 1.60, 0.0], [0.98, 1.78, 0.05], [0.98, 1.78, -0.05],
    [1.05, 1.70, 0.0]])
_HORSE35_PARENTS = [-1, 0, 1, 2, 3, 4, 5, 6, 4, 8, 9, 10, 4, 12, 13, 14, 0, 16, 17, 18, 0, 20, 21, 22, 2, 1, 4, 0,
                    0, 28, 29, 7, 7, 7, 7]
_HORSE35_RADII = [0.20, 0.20, 0.21, 0.20, 0.18, 0.11, 0.09, 0.08, 0.07, 0.06, 0.045, 0.04, 0.07, 0.06, 0.045, 0.04,
                  0.08, 0.065, 0.045, 0.04, 0.08, 0.065, 0.045, 0.04, 0.12, 0.12, 0.10, 0.10, 0.04, 0.03, 0.025, 0.04,
                  0.02, 0.02, 0.03]

NUM_VERTS = {'smpl': 6890, 'smplh': 6890, 'smplx': 10475, 'mano': 778, 'animal_horse': 3889}


def _bone_segments(pos, par, rad):
    """One segment per (joint, child) pair, plus a stub for leaves; the segment is owned by the joint."""
    nj = len(par)
    children = [[] for _ in range(nj)]
    for j in range(1, nj):
        children[par[j]].append(j)
    segs = []
    for j in range(nj):
        if children[j]:
            for c in children[j]:
                segs.append((j, pos[j], pos[c], rad[j]))
        else:
            d = pos[j] - pos[par[j]] if par[j] >= 0 else np.array([0, 1.0, 0])
            d = d / (np.linalg.norm(d) + 1e-12)
            segs.append((j, pos[j], pos[j] + d * max(1.6 * rad[j], 0.015), rad[j]))
    return segs


def _seg_dist(v, a, b):
    ab = b - a
    t = np.clip(((v - a) @ ab) / (ab @ ab + 1e-18), 0.0, 1.0)
    proj = a + t[:, None] * ab
    return np.linalg.norm(v - proj, axis=1), proj


def _sample_capsules(segs, n_total, rng, torso_joints=()):
    area = np.array([2 * np.pi * r * (np.linalg.norm(b - a) + r) for (_, a, b, r) in segs])
    share = area / area.sum() * n_total
    cnt = np.maximum(np.floor(share).astype(int), 10)
    while cnt.sum() > n_total:
        cnt[np.argmax(cnt)] -= 1
    rem = n_total - cnt.sum()
    order = np.argsort(-(share - np.floor(share)))
    for i in range(rem):
        cnt[order[i % len(order)]] += 1
    verts = []
    for (j, a, b, r), n in zip(segs, cnt):
        axis = b - a
        L = np.linalg.norm(axis)
        axis = axis / (L + 1e-12)
        ref = np.array([0.0, 0.0, 1.0]) if abs(axis[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
        e1 = np.cross(axis, ref)
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(axis, e1)
        u = (np.arange(n) + rng.uniform(0.2, 0.8, n)) / n
        phi = 2 * np.pi * ((np.arange(n) * 0.6180339887498949) % 1.0) + rng.uniform(-0.1, 0.1, n)
        r1, r2 = (1.25 * r, 0.8 * r) if j in torso_joints else (r, r)
        rr = 1.0 + 0.05 * rng.standard_normal(n)
        p = a[None] + (u * L)[:, None] * axis[None] \
            + (r1 * rr * np.cos(phi))[:, None] * e1[None] + (r2 * rr * np.sin(phi))[:, None] * e2[None]
        verts.append(p)
    return np.vstack(verts)


def _smooth_fields(verts, n_cols, std, rng, n_centres=24, width=0.18):
    idx = rng.choice(len(verts), size=n_centres, replace=False)
    d2 = ((verts[:, None, :] - verts[idx][None]) ** 2).sum(-1)
    phi = np.exp(-d2 / width ** 2)
    phi /= phi.sum(1, keepdims=True) + 1e-12
    z = rng.standard_normal((n_centres, n_cols))
    f = phi @ z
    return f * (std / (f.std() + 1e-12))


def make_body_model(model_type: str, n_verts: Optional[int] = None, n_betas: int = 24,
                    seed: int = SEED_MODEL) -> Dict:
    """Procedural body model in the reference's pickle format (SURVEY.md Appendix C)."""
    rng = np.random.default_rng(seed)
    pos, par, rad = skeleton(model_type)
    nj = len(par)
    V = n_verts or NUM_VERTS[model_type]
    segs = _bone_segments(pos, par, rad)
    n_eye = 0
    if model_type == 'smplx':
        n_eye = 1092 if V == 10475 else 0
        segs_body = [s for s in segs if s[0] not in (23, 24)]
    else:
        segs_body = segs
    torso = {'mano': (), 'animal_horse': (0, 1, 2, 3, 4)}.get(model_type, (0, 3, 6, 9))
    verts = _sample_capsules(segs_body, V - n_eye, rng, torso_joints=torso)
    verts = verts[rng.permutation(len(verts))]
    if n_eye:
        eyes = []
        for j in (23, 24):
            d = rng.standard_normal((n_eye // 2, 3))
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            eyes.append(pos[j][None] + 0.012 * d)
        verts = np.vstack([verts] + eyes)          # eyeballs are the tail block, like SMPL-X
    assert verts.shape == (V, 3)

    # skinning weights: top-4 of a Gaussian in the distance to each joint's bones
    dist = np.full((V, nj), np.inf)
    for (j, a, b, r) in segs:
        d, _ = _seg_dist(verts, a, b)
        dist[:, j] = np.minimum(dist[:, j], d)
    score = np.exp(-(dist / (0.6 * rad[None, :] + 0.01)) ** 2)
    top = np.argsort(-score, axis=1)[:, :4]
    W = np.zeros((V, nj))
    rows = np.arange(V)[:, None]
    W[rows, top] = np.take_along_axis(score, top, axis=1) + 1e-9
    W[W < 1e-3 * W.max(1, keepdims=True)] = 0.0
    W /= W.sum(1, keepdims=True)

    # joint regressor: least-norm affine combination of the 32 nearest vertices that hits the joint
    k = min(32, V)
    jr = np.zeros((nj, V))
    for j in range(nj):
        nn = np.argsort(((verts - pos[j]) ** 2).sum(1))[:k]
        B = np.vstack([verts[nn].T, np.ones(k)])
        w = B.T @ np.linalg.solve(B @ B.T + 1e-12 * np.eye(4), np.append(pos[j], 1.0))
        jr[j, nn] = w

    shapedirs = _smooth_fields(verts, 3 * n_betas, 5e-3, rng).reshape(V, 3, n_betas)
    shapedirs[:, :, 0] += 0.03 * (verts - verts.mean(0))          # a global-scale component
    posedirs = _smooth_fields(verts, 3 * 9 * (nj - 1), 2e-3, rng).reshape(V, 3, 9 * (nj - 1))

    kintree = np.vstack([np.array(par, dtype=np.int64), np.arange(nj, dtype=np.int64)])
    kintree = kintree.astype(np.uint32)            # root parent becomes 4294967295 as in the public files
    # faces (used by Stage I's surface term only): a fan of triangles around every vertex -- its nearest neighbours ordered by
    # angle in the tangent plane -- turned so that the normals point away from the nearest bone.  The fans overlap (this is
    # not a manifold; the reference's body models are watertight meshes), but they follow the sampled surface closely, so
    # distances to the mesh and their sign behave like on a real body.
    from sklearn.neighbors import NearestNeighbors
    kn = min(7, V)
    _, nbr = NearestNeighbors(n_neighbors=kn).fit(verts).kneighbors(verts)
    best = np.full(V, np.inf)
    proj = np.zeros_like(verts)
    for (_, a, b, _) in segs:
        dseg, pseg = _seg_dist(verts, a, b)
        upd = dseg < best
        best[upd] = dseg[upd]
        proj[upd] = pseg[upd]
    outward = verts - proj
    outward /= np.linalg.norm(outward, axis=1, keepdims=True) + 1e-12
    ref = np.where(np.abs(outward[:, :1]) < 0.9, np.array([[1.0, 0, 0]]), np.array([[0, 1.0, 0]]))
    t1 = np.cross(outward, ref)
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(outward, t1)
    rel = verts[nbr[:, 1:]] - verts[:, None, :]
    ang = np.arctan2((rel * t2[:, None, :]).sum(-1), (rel * t1[:, None, :]).sum(-1))
    order = np.argsort(ang, axis=1)
    ring = np.take_along_axis(nbr[:, 1:], order, axis=1)
    ang = np.take_along_axis(ang, order, axis=1)
    nxt = np.roll(ring, -1, axis=1)
    gap = np.mod(np.roll(ang, -1, axis=1) - ang, 2 * np.pi)
    keep = gap < 2.2                                   # no triangle across an open side of the fan
    centre = np.repeat(np.arange(V)[:, None], kn - 1, axis=1)
    faces = np.stack([centre[keep], ring[keep], nxt[keep]], axis=1)
    # a triangle found from several of its corners is kept once (duplicates with opposite orientation would make the SIGN of
    # the distance a coin toss); its orientation follows the mean outward direction of its three corners
    _, first = np.unique(np.sort(faces, axis=1), axis=0, return_index=True)
    faces = faces[np.sort(first)]
    flip = (np.cross(verts[faces[:, 1]] - verts[faces[:, 0]], verts[faces[:, 2]] - verts[faces[:, 0]]) * outward[faces].sum(1)).sum(1) < 0
    faces[flip] = faces[flip][:, [0, 2, 1]]
    faces = faces.astype(np.uint32)
    dd = {
        'v_template': verts, 'shapedirs': shapedirs, 'posedirs': posedirs, 'weights': W,
        'J_regressor': sp.csc_matrix(jr), 'kintree_table': kintree, 'f': faces,
        'bs_style': 'lbs', 'bs_type': 'lrotmin',
    }
    if model_type == 'mano':
        q, _ = np.linalg.qr(rng.standard_normal((45, 45)))
        dd['hands_components'] = q
        dd['hands_mean'] = 0.1 * rng.standard_normal(45)
    return dd


def make_hand_prior(seed: int = SEED_MODEL + 1) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    ql, _ = np.linalg.qr(rng.standard_normal((45, 45)))
    qr, _ = np.linalg.qr(rng.standard_normal((45, 45)))
    return {'componentsl': ql, 'componentsr': qr,
            'hands_meanl': 0.1 * rng.standard_normal(45), 'hands_meanr': 0.1 * rng.standard_normal(45)}


def make_body_prior(seed: int = SEED_MODEL + 2, n_comp: int = 8, dim: int = 69) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    means = 0.2 * rng.standard_normal((n_comp, dim))
    covars = np.zeros((n_comp, dim, dim))
    for k in range(n_comp):
        q, _ = np.linalg.qr(rng.standard_normal((dim, dim)))
        lam = np.exp(rng.uniform(np.log(0.05 ** 2), np.log(0.6 ** 2), dim))
        covars[k] = (q * lam) @ q.T
    weights = rng.dirichlet(np.ones(n_comp))
    return {'covars': covars, 'means': means, 'weights': weights}


def make_horse_prior(seed: int = SEED_MODEL + 4, dim: int = 105) -> Dict[str, np.ndarray]:
    """The horse pose prior's file layout (prior/horse_body_prior.py:41-47): 'pic' (a square root of the precision) and
    'mean_pose' over the pose without the root."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((dim, dim)))
    lam = np.exp(rng.uniform(np.log(1.0 / 0.6), np.log(1.0 / 0.08), dim))
    return {'pic': (q * lam) @ q.T, 'mean_pose': 0.1 * rng.standard_normal(dim)}


def make_dmpl(verts: np.ndarray, seed: int = SEED_MODEL + 3, n_dmpl: int = 8) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    V = len(verts)
    return {'eigvec': _smooth_fields(verts, 3 * n_dmpl, 3e-3, rng).reshape(V, 3, n_dmpl)}


# --------------------------------------------------------------------------------------
# marker layouts (SURVEY.md Appendix D) and latent markers (chmosh.py:57-80)
# --------------------------------------------------------------------------------------
def _fps(points: np.ndarray, n: int, rng) -> np.ndarray:
    sel = [int(rng.integers(len(points)))]
    d = ((points - points[sel[0]]) ** 2).sum(1)
    for _ in range(n - 1):
        i = int(np.argmax(d))
        sel.append(i)
        d = np.minimum(d, ((points - points[i]) ** 2).sum(1))
    return np.array(sel)


def make_layout(model: Dict, model_type: str, n_body: int, n_finger: int, seed: int = SEED_LAYOUT,
                hand_side: str = 'left', n_face: int = 0):
    """Returns (latent_labels, vids, marker_meta) with the reference's ordering
    (types sorted, labels sorted within type; marker_layout/edit_tools.py:136,148)."""
    rng = np.random.default_rng(seed)
    verts, W = model['v_template'], model['weights']
    nj = W.shape[1]
    dom = W.argmax(1)
    if model_type == 'mano':
        vids = _fps(verts, n_finger, rng)
        mtype = f'finger_{hand_side}'
        labels = [f'M{i:02d}' for i in range(n_finger)]
        groups = [(mtype, sorted(zip(labels, vids)))]
    else:
        n_hand = 15 if model_type in ('smplh', 'smplx') else 0
        first_hand = nj - 2 * n_hand
        body_mask = dom < first_hand
        if model_type == 'smplx':
            body_mask &= ~np.isin(dom, (22, 23, 24))
            body_mask[_pack.SMPLX_FIRST_EYEBALL_VID:] = False
        cand = np.nonzero(body_mask)[0]
        bsel = cand[_fps(verts[cand], n_body, rng)]
        extra = ['LBUM', 'RBUM', 'LKNI', 'RKNI']
        names = (STD46 + extra)[:n_body] if n_body > 41 else [l for l in STD46 if l not in ('LBAK', 'RBAK', 'T8', 'LMT1', 'RMT1')][:n_body]
        if len(names) < n_body:
            names += [f'B{i:02d}' for i in range(n_body - len(names))]
        groups = [('body', sorted(zip(names, bsel)))]
        if n_finger and n_hand:
            fl = FINGER6 if n_finger <= 6 else FINGER10
            fl = (fl + [f'FX{i}' for i in range(n_finger)])[:n_finger]
            for side, lo in (('left', first_hand), ('right', first_hand + n_hand)):
                cand = np.nonzero((dom >= lo) & (dom < lo + n_hand))[0]
                fsel = cand[_fps(verts[cand], n_finger, rng)]
                pref = 'L' if side == 'left' else 'R'
                groups.append((f'finger_{side}', sorted(zip([pref + n for n in fl], fsel))))
    if n_face and model_type == 'smplx':                 # markers on the head / jaw region, type 'face'
        cand = np.nonzero(np.isin(dom, (15, 22)))[0]
        cand = cand[cand < _pack.SMPLX_FIRST_EYEBALL_VID]
        fsel = cand[_fps(verts[cand], n_face, rng)]
        groups.append(('face', sorted(zip([f'FACE{i:02d}' for i in range(n_face)], fsel))))
    groups.sort(key=lambda g: g[0])
    labels, vids, mtypes = [], [], []
    for t, items in groups:
        for l, v in items:
            labels.append(l)
            vids.append(int(v))
            mtypes.append(t)
    type_names = sorted(set(mtypes))
    marker_meta = {
        'marker_vids': OrderedDict(zip(labels, vids)),
        'marker_type': OrderedDict(zip(labels, mtypes)),
        'marker_type_mask': OrderedDict((t, np.array([m == t for m in mtypes])) for t in type_names),
        'm2b_distance': {t: (0.0095 if t == 'body' else 0.0002) for t in type_names},
        'surface_model_type': model_type,
    }
    return labels, np.array(vids), marker_meta


def make_markers_latent(model: Dict, model_type: str, betas: np.ndarray, num_betas: int, vids, marker_meta):
    """v_shaped[vid] + outward direction * m2b (cf. chmosh.py:57-80; the direction is the vector from
    the nearest bone point to the vertex because the fixture has no face normals)."""
    v_shaped = model['v_template'] + model['shapedirs'][:, :, :num_betas].dot(betas[:num_betas])
    pos, par, rad = skeleton(model_type)
    segs = _bone_segments(pos, par, rad)
    pts = v_shaped[vids]
    best = np.full(len(pts), np.inf)
    proj = np.zeros_like(pts)
    for (_, a, b, _) in segs:
        d, p = _seg_dist(pts, a, b)
        upd = d < best
        best[upd] = d[upd]
        proj[upd] = p[upd]
    n = pts - proj
    n /= np.linalg.norm(n, axis=1, keepdims=True) + 1e-12
    m2b = np.array([marker_meta['m2b_distance'][t] for t in marker_meta['marker_type'].values()])
    return pts + n * m2b[:, None]


# --------------------------------------------------------------------------------------
# motion + observation synthesis
# --------------------------------------------------------------------------------------
def rodrigues_batch(rv: np.ndarray) -> np.ndarray:
    """Axis-angle (..., 3) -> rotation matrices (..., 3, 3)."""
    th = np.linalg.norm(rv, axis=-1, keepdims=True)
    small = th < 1e-8
    ths = np.where(small, 1.0, th)
    k = rv / ths
    K = np.zeros(rv.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2] = -k[..., 2], k[..., 1]
    K[..., 1, 0], K[..., 1, 2] = k[..., 2], -k[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -k[..., 1], k[..., 0]
    s, c = np.sin(th)[..., None], np.cos(th)[..., None]
    R = np.eye(3) + s * K + (1 - c) * (K @ K)
    # first-order form for tiny angles
    Ks = np.zeros_like(K)
    Ks[..., 0, 1], Ks[..., 0, 2] = -rv[..., 2], rv[..., 1]
    Ks[..., 1, 0], Ks[..., 1, 2] = rv[..., 2], -rv[..., 0]
    Ks[..., 2, 0], Ks[..., 2, 1] = -rv[..., 1], rv[..., 0]
    return np.where(small[..., None], np.eye(3) + Ks, R)


def rodrigues_inv_batch(R: np.ndarray) -> np.ndarray:
    """Rotation matrices (..., 3, 3) -> axis-angle (..., 3) with the angle in [0, pi] (away from pi: the skew part; near
    pi: the axis from the symmetric part)."""
    r = np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    s = 0.5 * np.linalg.norm(r, axis=-1)
    th = np.arctan2(s, (np.trace(R, axis1=-2, axis2=-1) - 1.0) * 0.5)
    out = np.where(th[..., None] < 1e-12, 0.5 * r, r * (th / np.maximum(2.0 * s, 1e-300))[..., None])
    near_pi = th > np.pi - 1e-3
    if near_pi.any():
        c = np.cos(th[near_pi])[:, None, None]
        B = (0.5 * (R[near_pi] + np.swapaxes(R[near_pi], -1, -2)) - c * np.eye(3)) / (1.0 - c)     # = u u^T
        k = np.argmax(np.diagonal(B, axis1=-2, axis2=-1), axis=-1)
        u = B[np.arange(len(B)), :, k]
        u /= np.linalg.norm(u, axis=-1, keepdims=True)
        u *= np.where((u * r[near_pi]).sum(-1) < 0, -1.0, 1.0)[:, None]
        out[near_pi] = u * th[near_pi][:, None]
    return out


def unwrap_axis_angle(rv: np.ndarray) -> np.ndarray:
    """Axis-angle rows (F, 3) of a rotation trajectory, each replaced by the equivalent rotation vector u (theta + 2 pi n)
    nearest to the row before: the continuous trajectory an iterative solver warm-started from the previous frame
    follows (|theta| > pi once it has turned past pi)."""
    out = np.array(rv, dtype=np.float64)
    for f in range(1, len(out)):
        th = np.linalg.norm(out[f])
        if th < 1e-12:
            continue
        u = out[f] / th
        out[f] = u * (th + 2 * np.pi * np.round((u @ out[f - 1] - th) / (2 * np.pi)))
    return out


def make_motion(p: _pack.StageIIPack, n_frames: int, seed: int, fps: float = 120.0,
                body_amp: float = 0.35, finger_amp: float = 0.25, root_yaw=None):
    """Smooth reduced-pose / translation / DMPL trajectories (SURVEY.md 8(d) "Motion").  ``root_yaw``: a turn of the
    whole body about the up (y) axis -- (yaw_start, yaw_end) rad, linear in time, or one yaw per frame -- composed in
    front of the small root motion; the root is then the continuous axis-angle trajectory (``unwrap_axis_angle``).
    None keeps the random draws and the motion as they are."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_frames) / fps
    P = p.p_red
    pose = np.zeros((n_frames, P))
    for i in range(P):
        amp = body_amp if i < p.body_dof else finger_amp
        if i < 3:
            amp = 0.25
        a = rng.uniform(0.2, 1.0, 3) * amp / 3.0
        f = rng.uniform(0.2, 2.0, 3)
        ph = rng.uniform(0, 2 * np.pi, 3)
        pose[:, i] = (a[None] * np.sin(2 * np.pi * f[None] * t[:, None] + ph[None])).sum(1) + rng.normal(0, 0.05 * amp)
    if p.model_type in ('smpl', 'smplh', 'smplx', 'animal_horse'):
        pose[:, 30:36] *= 0.0            # toes are frozen in Stage II unless optimize_toes
    if p.model_type == 'animal_horse':
        pose[:, 84:] = 0.0               # tail, mouth and ears are never optimised (chmosh.py:572-573)
        pose[:, 3:84] *= 0.6
    if p.model_type == 'smplx':
        if p.face_hi > p.face_lo:
            pose[:, 69:75] = 0.0         # eyes are never optimised; the jaw is, with optimize_face
            pose[:, 66:69] *= 0.3
        else:
            pose[:, 66:75] = 0.0         # jaw / eyes are not optimised without optimize_face
    trans = np.stack([0.5 * np.sin(2 * np.pi * 0.1 * t + 0.3), 0.03 * np.sin(2 * np.pi * 1.1 * t) + 0.9,
                      0.8 * t / max(t[-1], 1e-9) * min(1.0, t[-1]) + 0.2 * np.sin(2 * np.pi * 0.07 * t)], axis=1)
    dm = np.zeros((n_frames, p.n_dmpl))
    if p.n_dmpl:
        e = rng.standard_normal((n_frames, p.n_dmpl))
        rho = 0.97
        dm[0] = 0.5 * e[0]
        for k in range(1, n_frames):
            dm[k] = rho * dm[k - 1] + np.sqrt(1 - rho ** 2) * 0.5 * e[k]
    if root_yaw is not None:
        yaw = np.asarray(root_yaw, dtype=np.float64)
        if yaw.shape == (2,) and n_frames != 2:
            yaw = np.linspace(yaw[0], yaw[1], n_frames)
        if yaw.shape != (n_frames,):
            raise ValueError(f'root_yaw: (start, end) or {n_frames} values')
        R = rodrigues_batch(yaw[:, None] * np.array([0.0, 1.0, 0.0])) @ rodrigues_batch(pose[:, :3])
        pose[:, :3] = unwrap_axis_angle(rodrigues_inv_batch(R))
    return pose, trans, dm


def forward_markers(p: _pack.StageIIPack, pose: np.ndarray, trans: np.ndarray,
                    dmpl: Optional[np.ndarray] = None, block: int = 256) -> np.ndarray:
    """Simulated markers F x M x 3 for reduced poses (vectorised over frames, selected vertices only)."""
    F = pose.shape[0]
    out = np.zeros((F, p.n_markers, 3))
    nj, S = p.n_joints, 3 * p.n_markers
    wj = np.where(p.w_joint < 0, 0, p.w_joint)
    for lo in range(0, F, block):
        hi = min(F, lo + block)
        th, tr = pose[lo:hi], trans[lo:hi]
        B = hi - lo
        full = np.zeros((B, p.p_full))
        full[:, :p.body_dof] = th[:, :p.body_dof]
        if p.n_hand_full:
            full[:, p.body_dof:] = p.hands_mean[None] + th[:, p.body_dof:] @ p.hand_comps
        R = rodrigues_batch(full.reshape(B, nj, 3))
        pf = (R[:, 1:] - np.eye(3)).reshape(B, nj - 1, 9)
        vsh = np.broadcast_to(p.v0[None], (B, S, 3)).copy()
        jp = np.broadcast_to(p.j0[None], (B, nj, 3)).copy()
        if p.n_dmpl and dmpl is not None:
            d = dmpl[lo:hi]
            vsh += np.einsum('scd,bd->bsc', p.sd, d)
            jp += np.einsum('jcd,bd->bjc', p.jd, d)
        vp = vsh + np.einsum('jrn,bjn->br', p.pd, pf).reshape(B, S, 3)
        Rg = np.zeros((B, nj, 3, 3))
        tg = np.zeros((B, nj, 3))
        Rg[:, 0], tg[:, 0] = R[:, 0], jp[:, 0]
        for j in range(1, nj):
            a = p.parents[j]
            Rg[:, j] = Rg[:, a] @ R[:, j]
            tg[:, j] = tg[:, a] + np.einsum('bcd,bd->bc', Rg[:, a], jp[:, j] - jp[:, a])
        v = np.zeros((B, S, 3))
        for i in range(p.kw):
            ji = wj[:, i]
            pij = np.einsum('bscd,bsd->bsc', Rg[:, ji], vp - jp[:, ji]) + tg[:, ji]
            v += p.w_val[None, :, i, None] * pij
        v += tr[:, None, :]
        v = v.reshape(B, p.n_markers, 3, 3)
        e1 = v[:, :, 1] - v[:, :, 0]
        e2 = v[:, :, 2] - v[:, :, 0]
        f1 = e1 / np.linalg.norm(e1, axis=-1, keepdims=True)
        n = np.cross(e1, e2)
        f2 = n / np.linalg.norm(n, axis=-1, keepdims=True)
        f3 = np.cross(f1, f2)
        k = p.coefs[None]
        out[lo:hi] = v[:, :, 0] + k[..., 0:1] * f1 + k[..., 1:2] * f2 + k[..., 2:3] * f3
    return out


# --------------------------------------------------------------------------------------
# configs (BASELINE.json) and case writer
# --------------------------------------------------------------------------------------
CONFIGS = {
    # name: model_type, frames, n_body, n_finger, fingers, dynamics
    'C1': dict(model_type='smpl', frames=12, n_body=41, n_finger=0, optimize_fingers=False, optimize_dynamics=False, mocap_ext='c3d'),
    'C2': dict(model_type='smplh', frames=500, n_body=41, n_finger=6, optimize_fingers=True, optimize_dynamics=False, mocap_ext='npz'),
    'C3': dict(model_type='smplx', frames=4000, n_body=47, n_finger=10, optimize_fingers=True, optimize_dynamics=True, mocap_ext='npz'),
    'C4': dict(model_type='mano', frames=2000, n_body=0, n_finger=20, optimize_fingers=True, optimize_dynamics=False, mocap_ext='npz'),
    'C5': dict(model_type='smplh', frames=4000, n_body=41, n_finger=6, optimize_fingers=True, optimize_dynamics=False, mocap_ext='npz'),
    # widening row (SURVEY.md 8(f-4)): SMPL-X with face markers, jaw + expression coefficients free in Step 2
    'CF': dict(model_type='smplx', frames=200, n_body=41, n_finger=6, n_face=12, optimize_fingers=True, optimize_dynamics=False,
               optimize_face=True, mocap_ext='npz'),
    # (new configurations go last: the motion seed depends on the position)
    # the one animal variant whose Stage II runs in the reference
    'CH': dict(model_type='animal_horse', frames=60, n_body=36, n_finger=0, optimize_fingers=False, optimize_dynamics=False, mocap_ext='npz'),
}


# make_case arguments of a model with the reference's SMPL-X face layout (moshpp_conf.yaml: betas_expr_start_id 300,
# num_expressions 80; SMPL-X files carry 400 shape components)
REFERENCE_FACE = dict(n_betas=400, expr_start=300, num_expressions=80)

from .cfg import AttrDict, STAGEII_WEIGHTS, default_cfg  # noqa: E402,F401


def make_case(out_dir: str, config: str = 'C2', *, frames: Optional[int] = None, n_verts: Optional[int] = None,
              seq_idx: int = 0, noise_mm: float = 1.0, dropout: float = 0.03, hand_side: str = 'left',
              write_mocap: bool = True, reuse_model: bool = True, model_seed: int = 0, n_betas: int = 24,
              expr_start: int = 16, num_expressions: int = 8, root_yaw=None) -> Dict:
    """Writes one synthetic Stage-II case (model, priors, mocap file) and returns everything
    ``mosh_stageii`` needs plus the ground truth.  ``seq_idx`` picks the shape (and with it the latent markers) and the
    motion; ``model_seed`` > 0 writes and uses a second model file of the same family and size (another template, shape
    space and joint regressor; e.g. the other gender's model).  ``n_betas``: shape components of the model file;
    ``expr_start`` / ``num_expressions``: the expression components of the configurations with ``optimize_face``
    (``REFERENCE_FACE`` is the layout of the reference's SMPL-X face setup); ``root_yaw``: a turn of the whole body about
    the up axis (``make_motion``)."""
    c = dict(CONFIGS[config])
    mt = c['model_type']
    F = int(frames or c['frames'])
    os.makedirs(out_dir, exist_ok=True)
    tag = (f'{mt}_{n_verts or NUM_VERTS[mt]}' + (f'_{hand_side}' if mt == 'mano' else '') + (f'_m{model_seed}' if model_seed else '')
           + (f'_b{n_betas}' if n_betas != 24 else ''))
    model_fname = os.path.join(out_dir, f'model_{tag}.pkl')
    hand_prior_fname = os.path.join(out_dir, 'pose_hand_prior.npz')
    body_prior_fname = os.path.join(out_dir, 'pose_body_prior.pkl')
    dmpl_fname = os.path.join(out_dir, f'dmpl_{tag}.pkl')
    if reuse_model and os.path.exists(model_fname):
        with open(model_fname, 'rb') as f:
            model = pickle.load(f)
    else:
        model = make_body_model(mt, n_verts=n_verts, n_betas=n_betas,
                                seed=SEED_MODEL + (7 if hand_side == 'right' else 0) + 1000 * model_seed)
        with open(model_fname, 'wb') as f:
            pickle.dump(model, f, protocol=pickle.HIGHEST_PROTOCOL)
    if not os.path.exists(hand_prior_fname):
        np.savez(hand_prior_fname, **make_hand_prior())
    if mt == 'animal_horse':
        body_prior_fname = os.path.join(out_dir, 'pose_body_prior_horse.pkl')
        if not os.path.exists(body_prior_fname):
            with open(body_prior_fname, 'wb') as f:
                pickle.dump(make_horse_prior(), f, protocol=pickle.HIGHEST_PROTOCOL)
    elif not os.path.exists(body_prior_fname):
        with open(body_prior_fname, 'wb') as f:
            pickle.dump(make_body_prior(), f, protocol=pickle.HIGHEST_PROTOCOL)
    if c['optimize_dynamics'] and not os.path.exists(dmpl_fname):
        with open(dmpl_fname, 'wb') as f:
            pickle.dump(make_dmpl(model["v_template"]), f, protocol=pickle.HIGHEST_PROTOCOL)

    rng = np.random.default_rng(SEED_MODEL + 100 + seq_idx)
    betas = np.zeros(model['shapedirs'].shape[-1])
    betas[:16] = rng.standard_normal(16)
    labels, vids, marker_meta = make_layout(model, mt, c['n_body'], c['n_finger'], hand_side=hand_side, n_face=c.get('n_face', 0))
    markers_latent = make_markers_latent(model, mt, betas, 16, vids, marker_meta)

    cfg = default_cfg(**{
        'surface_model.type': mt, 'surface_model.fname': model_fname, 'surface_model.dmpl_fname': dmpl_fname,
        'moshpp.pose_body_prior_fname': body_prior_fname, 'moshpp.pose_hand_prior_fname': hand_prior_fname,
        'moshpp.optimize_fingers': c['optimize_fingers'], 'moshpp.optimize_dynamics': c['optimize_dynamics'],
        'moshpp.verbosity': 0,
    })
    face = bool(c.get('optimize_face', False))
    if face:                 # by default the model has 24 shape components: 16 betas, then 8 used as expressions
        cfg.moshpp.optimize_face = True
        cfg.surface_model.betas_expr_start_id = expr_start
        cfg.surface_model.num_expressions = num_expressions

    sm = _pack.load_surface_model(model_fname, pose_hand_prior_fname=hand_prior_fname,
                                  use_hands_mean=cfg.surface_model.use_hands_mean,
                                  dof_per_hand=cfg.surface_model.dof_per_hand, surface_model_type=mt)
    prior = None
    if mt == 'animal_horse':
        prior = _pack.create_horse_body_prior(body_prior_fname)
    elif mt != 'mano':
        prior = _pack.create_gmm_body_prior(body_prior_fname, exclude_hands=mt in ('smplh', 'smplx'))
    dm_dirs = None
    if c['optimize_dynamics']:
        with open(dmpl_fname, 'rb') as f:
            dm_dirs = pickle.load(f)['eigvec']
    pk = _pack.build_pack(sm, betas, markers_latent, num_betas=16, prior=prior, dmpl_dirs=dm_dirs,
                          num_dmpls=8 if c['optimize_dynamics'] else 0,
                          optimize_fingers=c['optimize_fingers'], optimize_face=face,
                          expr_start=expr_start if face else 0, num_expressions=num_expressions if face else 0)
    cfg_idx = list(CONFIGS).index(config)
    pose, trans, dm = make_motion(pk, F, seed=SEED_MOTION + cfg_idx + 1000 * seq_idx, root_yaw=root_yaw)
    if not c['optimize_fingers'] and pk.n_hand_red:
        pose[:, pk.body_dof:] = 0.0
    mk = forward_markers(pk, pose, trans, dm if pk.n_dmpl else None)
    nrng = np.random.default_rng(SEED_NOISE + seq_idx)
    obs = mk + nrng.normal(0.0, noise_mm * 1e-3, mk.shape)
    drng = np.random.default_rng(SEED_DROPOUT + seq_idx)
    vis = np.ones((F, pk.n_markers), dtype=bool)
    if dropout > 0:
        for m in range(pk.n_markers):
            missing = 0
            while missing < dropout * F:
                L = int(drng.integers(5, 51)) if F >= 100 else int(drng.integers(1, max(2, F // 10) + 1))
                s = int(drng.integers(0, max(1, F - 1)))
                vis[s:s + L, m] = False
                missing += L
    # mocap file: other label order, two distractor channels, millimetres, missing = NaN
    perm = np.random.default_rng(SEED_LAYOUT + 1).permutation(pk.n_markers)
    file_labels = [labels[i] for i in perm] + ['*57', 'EXTRA1']
    data = np.full((F, pk.n_markers + 2, 3), np.nan)
    data[:, :pk.n_markers] = np.where(vis[:, perm, None], obs[:, perm], np.nan) * 1000.0
    data[:, -1] = 1000.0 * (trans + 0.3)
    side = f'_{hand_side}' if mt == 'mano' else ''
    # (a model with another shape space, or other expressions, synthesises other observations: a file of its own)
    size = f'_b{n_betas}' if n_betas != 24 else ''
    size += f'_e{expr_start}x{num_expressions}' if face and (expr_start, num_expressions) != (16, 8) else ''
    if root_yaw is not None:
        size += '_yaw' + hashlib.blake2b(np.asarray(root_yaw, dtype=np.float64).tobytes(), digest_size=4).hexdigest()
    mocap_fname = os.path.join(out_dir, f'mocap_{config}{side}{size}_{seq_idx:02d}_{F}.{c["mocap_ext"]}')
    if write_mocap:
        if c['mocap_ext'] == 'npz':
            np.savez(mocap_fname, markers=data, labels=np.array(file_labels), frame_rate=120.0)
        else:
            from .c3d_io import write_c3d
            write_c3d(mocap_fname, data, file_labels, frame_rate=120.0)
    cfg.mocap.fname = mocap_fname
    return dict(cfg=cfg, mocap_fname=mocap_fname, markers_latent=markers_latent, latent_labels=labels,
                betas=betas, marker_meta=marker_meta, pack=pk, gt_pose=pose, gt_trans=trans, gt_dmpl=dm,
                gt_markers=mk, obs=obs, vis=vis, model=model, config=c)


from .stagei import write_marker_layout  # noqa: E402,F401  (re-exported: the fixtures write their layouts with it)


def make_subject(out_dir: str, config: str = 'C2', frames=(1000, 2000), **kw):
    """Several captures of ONE synthetic subject (one shape, one set of latent markers): a case of ``sum(frames)`` frames
    (``make_case``, npz configurations) whose capture file is cut into consecutive captures of ``frames[k]`` frames.
    ``seq_idx`` (shape, latent markers and motion) and ``model_seed`` (a second model file) of ``make_case`` make other
    subjects.  Returns (the case, the capture file names)."""
    case = make_case(out_dir, config, frames=int(sum(frames)), **kw)
    if not case['mocap_fname'].endswith('.npz'):
        raise ValueError(f'{config}: make_subject cuts npz captures only')
    z = np.load(case['mocap_fname'])
    stem = os.path.splitext(case['mocap_fname'])[0]
    fnames, f0 = [], 0
    for k, F in enumerate(frames):
        fn = f'{stem}_take{k:02d}_{int(F)}.npz'
        np.savez(fn, markers=z['markers'][f0:f0 + int(F)], labels=z['labels'], frame_rate=z['frame_rate'])
        fnames.append(fn)
        f0 += int(F)
    return case, fnames
