"""Once-per-sequence host preprocessing for the device solver.

Everything here runs once per (subject model, betas, marker layout) and is index / layout
work: load the body-model pickle in the reference's on-disk format, attach the latent markers
to the canonical mesh, gather the <= 3*M vertices the markers touch and lay their constants out
for the kernels (DESIGN.md "Data layout in HBM").  The per-frame arithmetic (SMPL forward,
Jacobians, priors, dog-leg) lives only in ``csrc/`` -- there is no CPU solver in this package.

Reference behaviour restated here (file:line under /root/reference/src/moshpp):
  * model parametrisation / hand PCA ........ models/smpl_fast_derivatives.py:52-166,194-204
  * marker attachment (TransformedCoeffs) .... transformed_lm.py:45-113
  * GMM body prior constants ................. prior/gmm_prior_ch.py:107-134, prior/dog_body_prior.py:53-87
  * pose-id partitions, toes, fingers ........ chmosh.py:548-571,645-647,676-692
"""
from __future__ import annotations

import os
import pickle
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

# SMPL-X eyeball vertices are excluded from marker attachment (transformed_lm.py:47-50,67-70).
# The reference reads them from support_data/smplx_eyeballs.npz; that file holds exactly the
# tail block 9383..10474 (checked when this module was written), so the candidate set is 0..9382.
SMPLX_NUM_VERTS = 10475
SMPLX_FIRST_EYEBALL_VID = 9383

MODEL_TYPE_BY_NJOINT_PARMS = {69: 'smpl', 153: 'smplh', 162: 'smplx', 45: 'mano'}


# --------------------------------------------------------------------------------------
# model loading (reference: models/smpl_fast_derivatives.py:52-166)
# --------------------------------------------------------------------------------------
@dataclass
class SurfaceModel:
    model_type: str
    v_template: np.ndarray      # V x 3
    shapedirs: np.ndarray       # V x 3 x nbeta_model
    posedirs: np.ndarray        # V x 3 x 9(nJ-1)
    weights: np.ndarray         # V x nJ
    J_regressor: np.ndarray     # nJ x V dense (converted from sparse)
    parents: np.ndarray         # nJ, -1 for the root
    body_dof: int               # leading full-pose entries that map 1:1 to the reduced pose
    hand_comps: np.ndarray      # n_hand_red x n_hand_full   ("selected_components")
    hands_mean: np.ndarray      # n_hand_full
    faces: Optional[np.ndarray] = None

    @property
    def n_joints(self) -> int:
        return self.weights.shape[1]

    @property
    def p_full(self) -> int:
        return 3 * self.n_joints

    @property
    def p_red(self) -> int:
        return self.body_dof + self.hand_comps.shape[0]


def _dense_regressor(jreg) -> np.ndarray:
    if hasattr(jreg, 'toarray'):
        return np.asarray(jreg.toarray(), dtype=np.float64)
    if hasattr(jreg, 'row') and hasattr(jreg, 'col'):  # coo-like struct from old pickles
        out = np.zeros(jreg.shape, dtype=np.float64)
        np.add.at(out, (np.asarray(jreg.row), np.asarray(jreg.col)), np.asarray(jreg.data))
        return out
    return np.asarray(jreg, dtype=np.float64)


class _ChLeaf:
    """What a ``chumpy.ch.Ch`` leaf of a public body-model pickle becomes when chumpy is not installed.  The released
    SMPL / SMPL-H / MANO files store ``v_template``, ``shapedirs``, ``posedirs``, ``weights``, ``J`` as pickled chumpy
    objects (the reference reads them through chumpy, smpl_fast_derivatives.py:48,149-166); a leaf's state is a dict whose
    ``x`` entry is the array.  Nothing of chumpy is evaluated: anything that is not a plain leaf is refused."""

    def __setstate__(self, state):
        self.__dict__.update(state if isinstance(state, dict) else {})

    def __array__(self, dtype=None, copy=None):
        if 'x' not in self.__dict__:
            raise TypeError('pickled chumpy object without an array payload (not a leaf): install chumpy to read this file')
        a = np.asarray(self.__dict__['x'])
        return a.astype(dtype) if dtype is not None else a

    @property
    def r(self):
        return self.__array__()


class _ModelUnpickler(pickle.Unpickler):
    """pickle.load for body-model / prior files written by the reference's environment, without that environment:
    chumpy classes resolve to chumpy when it is importable and to ``_ChLeaf`` otherwise; scipy.sparse classes pickled under
    their old private module paths (``scipy.sparse.csc.csc_matrix`` ...) resolve to the public ones."""

    def find_class(self, module, name):
        top = module.split('.')[0]
        if top == 'chumpy':
            try:
                return super().find_class(module, name)
            except (ImportError, AttributeError):
                return _ChLeaf
        if module.startswith('scipy.sparse.'):
            try:
                return super().find_class(module, name)
            except (ImportError, AttributeError):
                import scipy.sparse
                return getattr(scipy.sparse, name)
        return super().find_class(module, name)


def load_reference_pickle(fname: str):
    """A pickle of the reference's world (python-2 ``latin-1`` strings, chumpy leaves, old scipy paths) as plain data:
    every chumpy value of a top-level dict is replaced by its array."""
    with open(fname, 'rb') as f:
        dd = _ModelUnpickler(f, encoding='latin-1').load()
    if isinstance(dd, dict):
        for k, v in list(dd.items()):
            if not isinstance(v, np.ndarray) and hasattr(v, 'r') and not hasattr(v, 'toarray'):
                dd[k] = np.asarray(v.r)
    return dd


_MODEL_FILE_CACHE: 'OrderedDict[tuple, dict]' = OrderedDict()


def _read_model_pickle(fname: str) -> dict:
    """The unpickled body-model file, kept for the (path, mtime, size) it was read from: a subject's sequences (and all
    subjects of one model family) share the 80-300 MB file, and unpickling it costs more than solving a sequence.  The
    entry is dropped as soon as the file changes; at most two models are kept.  The arrays are never written to."""
    st = os.stat(fname)
    key = (os.path.realpath(fname), st.st_mtime_ns, st.st_size)
    dd = _MODEL_FILE_CACHE.get(key)
    if dd is None:
        dd = load_reference_pickle(fname)
        _MODEL_FILE_CACHE[key] = dd
        while len(_MODEL_FILE_CACHE) > 2:
            _MODEL_FILE_CACHE.popitem(last=False)
    else:
        _MODEL_FILE_CACHE.move_to_end(key)
    return dd


def clear_file_cache():
    _MODEL_FILE_CACHE.clear()


def load_surface_model(surface_model_fname: str,
                       pose_hand_prior_fname: Optional[str] = None,
                       use_hands_mean: bool = False,
                       dof_per_hand: int = 12,
                       v_template: Optional[np.ndarray] = None,
                       surface_model_type: Optional[str] = None) -> SurfaceModel:
    """Same inputs and model-type rules as the reference loader (smpl_fast_derivatives.py:52-145)."""
    if not str(surface_model_fname).endswith('.pkl'):
        raise ValueError('surface_model_fname could only be a pkl file.')
    dd = _read_model_pickle(str(surface_model_fname))

    posedirs = np.asarray(dd['posedirs'], dtype=np.float64)
    njoint_parms = posedirs.shape[2] // 3
    model_type = surface_model_type or MODEL_TYPE_BY_NJOINT_PARMS[njoint_parms]

    if dd.get('bs_style', 'lbs') != 'lbs':
        raise AssertionError("bs_style must be 'lbs'")  # smpl_fast_derivatives.py:176

    kintree = np.asarray(dd['kintree_table'])
    parents = kintree[0].astype(np.int64).copy()
    parents[0] = -1
    parents[parents > len(parents)] = -1  # uint32(-1) root marker of the public pickles

    if model_type in ('smplx', 'smplh'):
        body_dof = njoint_parms - 90 + 3
        if pose_hand_prior_fname is None or not str(pose_hand_prior_fname).endswith('.npz'):
            raise AssertionError('pose_hand_prior_fname (.npz) is required for smplh/smplx')
        hp = np.load(pose_hand_prior_fname)
        cl = np.asarray(hp['componentsl'], dtype=np.float64)
        cr = np.asarray(hp['componentsr'], dtype=np.float64)
        ml = np.asarray(hp['hands_meanl'], dtype=np.float64) if use_hands_mean else np.zeros(cl.shape[1])
        mr = np.asarray(hp['hands_meanr'], dtype=np.float64) if use_hands_mean else np.zeros(cr.shape[1])
        zl = np.zeros_like(cl[:dof_per_hand])
        zr = np.zeros_like(cr[:dof_per_hand])
        comps = np.vstack((np.hstack((cl[:dof_per_hand], zl)), np.hstack((zr, cr[:dof_per_hand]))))
        hands_mean = np.concatenate((ml, mr))
    elif model_type == 'mano':
        body_dof = 3
        hc = np.asarray(dd['hands_components'], dtype=np.float64)
        # the flag is inverted for MANO in the reference (smpl_fast_derivatives.py:114)
        hands_mean = np.zeros(hc.shape[1]) if use_hands_mean else np.asarray(dd['hands_mean'], dtype=np.float64)
        comps = hc[:dof_per_hand].copy()
    else:
        body_dof = njoint_parms + 3
        comps = np.zeros((0, 0))
        hands_mean = np.zeros(0)

    vt = np.asarray(dd['v_template'], dtype=np.float64) if v_template is None else np.asarray(v_template, np.float64)
    model = SurfaceModel(
        model_type=model_type,
        v_template=vt,
        shapedirs=np.asarray(dd['shapedirs'], dtype=np.float64),
        posedirs=posedirs,
        weights=np.asarray(dd['weights'], dtype=np.float64),
        J_regressor=_dense_regressor(dd['J_regressor']),
        parents=parents,
        body_dof=int(body_dof),
        hand_comps=np.ascontiguousarray(comps),
        hands_mean=np.ascontiguousarray(hands_mean),
        faces=np.asarray(dd['f']) if 'f' in dd else None,
    )
    assert model.body_dof + model.hands_mean.shape[0] == model.p_full, \
        f'pose layout mismatch: {model.body_dof}+{model.hands_mean.shape[0]} != {model.p_full}'
    assert np.all(model.parents[1:] < np.arange(1, model.n_joints)), 'kintree must be topologically ordered'
    return model


# --------------------------------------------------------------------------------------
# marker attachment (reference: transformed_lm.py:59-113)
# --------------------------------------------------------------------------------------
def _nrm(x: np.ndarray) -> np.ndarray:
    with np.errstate(invalid='ignore', divide='ignore'):
        return x / np.sqrt(np.sum(x ** 2, axis=1)).reshape((-1, 1))


def attach_markers(can_verts: np.ndarray, markers_latent: np.ndarray):
    """8-NN local frames of the latent markers on the canonical mesh.

    Returns (closest M x 3 int64, coefs M x 3): marker = v[c0] + k1 f1 + k2 f2 + k3 f3.
    """
    can_verts = np.asarray(can_verts, dtype=np.float64)
    markers_latent = np.asarray(markers_latent, dtype=np.float64)
    cand = can_verts[:SMPLX_FIRST_EYEBALL_VID] if len(can_verts) == SMPLX_NUM_VERTS else can_verts
    # brute-force L2 8-NN, distance-sorted like sklearn's kd_tree query.  Axis by axis: the same squares added in the same
    # order as ((m - v) ** 2).sum(-1), without the M x V x 3 temporary (four times faster; Stage I attaches per evaluation)
    ct = np.ascontiguousarray(cand.T)
    d = markers_latent[:, 0, None] - ct[0][None, :]
    d2 = d * d
    d = markers_latent[:, 1, None] - ct[1][None, :]
    d2 += d * d
    d = markers_latent[:, 2, None] - ct[2][None, :]
    d2 += d * d
    k = min(8, cand.shape[0])
    part = np.argpartition(d2, k - 1, axis=1)[:, :k]
    order = np.argsort(np.take_along_axis(d2, part, axis=1), axis=1, kind='stable')
    closest = np.take_along_axis(part, order, axis=1).astype(np.int64)

    diff = markers_latent - can_verts[closest[:, 0]]
    e1 = can_verts[closest[:, 1]] - can_verts[closest[:, 0]]
    e2 = can_verts[closest[:, 2]] - can_verts[closest[:, 0]]
    f1 = _nrm(e1)
    nn = 3
    # collinear fallback: the reference swaps the third neighbour for *all* markers at once
    # (transformed_lm.py:94-100); its loop bound is closest.shape[0], ours is the 8 columns that exist.
    while np.isnan(_nrm(np.cross(e1, e2)).sum()) and nn < closest.shape[1]:
        e2 = can_verts[closest[:, nn]] - can_verts[closest[:, 0]]
        nn += 1
    closest[:, 2] = closest[:, nn - 1]
    f2 = _nrm(np.cross(e1, e2))
    if np.isnan(f2).any():
        raise ValueError('marker attachment failed: nearest canonical vertices are collinear')
    f3 = np.cross(f1, f2)
    coefs = np.stack([(diff * f1).sum(1), (diff * f2).sum(1), (diff * f3).sum(1)], axis=1)
    return np.ascontiguousarray(closest[:, :3]), np.ascontiguousarray(coefs)


# --------------------------------------------------------------------------------------
# GMM max-mixture body prior constants (reference: prior/gmm_prior_ch.py:107-134)
# --------------------------------------------------------------------------------------
@dataclass
class BodyPrior:
    means: np.ndarray      # K x D
    Q: np.ndarray          # K x D x D,  Q_k = 0.5 * inv(cov_k)  (= 0.5 * L_k L_k^T of the reference)
    neglogw: np.ndarray    # K,  -log(w_k) with the reference's normalisation


# joint-angle term of the horse model (prior/horse_body_prior.py:56-71): pose ids of the four legs' bend angles, all signs +1
HORSE_JANGLES_IDS = np.array([6, 7, 8, 11, 12, 13, 20, 21, 22, 25, 26, 27], dtype=np.int32)
HORSE_JANGLES_SIGNS = np.ones(12)


def create_horse_body_prior(pose_body_prior_fname: str) -> BodyPrior:
    """smal_horse_prior (prior/horse_body_prior.py:40-53, tail / mouth / ears disabled): r = (pose[3:84] - mean) . pic, i.e.
    one component with Q = pic pic^T and no weight constant."""
    res = load_reference_pickle(pose_body_prior_fname)
    P = np.asarray(res['pic'], dtype=np.float64)[:81, :81]
    mu = np.asarray(res['mean_pose'], dtype=np.float64)[:81]
    return BodyPrior(means=np.ascontiguousarray(mu[None]), Q=np.ascontiguousarray((P @ P.T)[None]), neglogw=np.zeros(1))


# SMAL dog (prior/dog_body_prior.py:56-58, chmosh.py:574-579): the joints its pose prior and Stage II see -- not 0 (the
# root, optimised on its own), 2, 6 and 29; their pose ids in this order (93 of the 105)
DOG_BODY_JOINTS = (1, 3, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28,
                   30, 31, 32, 33, 34)
DOG_BODY_IDS = np.array([3 * j + c for j in DOG_BODY_JOINTS for c in range(3)], dtype=np.int32)


def create_dog_body_prior(pose_body_prior_fname: str) -> BodyPrior:
    """MaxMixtureDog.get_gmm_prior (prior/dog_body_prior.py:53-87): the mixture of 'gmm_covs' / 'gmm_means' / 'gmm_weights'
    restricted to DOG_BODY_IDS, with MaxMixtureComplete's residual as for SMPL (gmm_prior_ch.py:42-104).

    The weight constant -log(w_k / ((2 pi)^(D/2) sqrt(det S_k) / min_j sqrt(det S_j))) is computed in the log domain:
    -log w_k + (D/2) log 2 pi + (logdet S_k - min_j logdet S_j) / 2.  That is the reference's value whenever the determinants
    are representable; at D = 93 a covariance with per-axis variances near 1e-4 has det = 0 in float64, where the direct form
    gives 0 / 0.  A covariance that is not positive definite raises ValueError (the reference asserts the opposite of what its
    message says, dog_body_prior.py:78-79, and so refuses every valid prior)."""
    gmm = load_reference_pickle(pose_body_prior_fname)
    ids = DOG_BODY_IDS
    covars = np.asarray(gmm['gmm_covs'], dtype=np.float64)[:, :, ids][:, ids]
    means = np.asarray(gmm['gmm_means'], dtype=np.float64)[:, ids]
    weights = np.asarray(gmm['gmm_weights'], dtype=np.float64).ravel()
    D = len(ids)
    logdets = np.zeros(len(covars))
    for k, c in enumerate(covars):
        try:
            np.linalg.cholesky(c)
        except np.linalg.LinAlgError:
            raise ValueError(f'dog pose prior {pose_body_prior_fname}: the covariance of component {k} is not positive '
                             f'definite') from None
        logdets[k] = np.linalg.slogdet(c)[1]
    precs = np.stack([np.linalg.inv(c) for c in covars])
    neglogw = -np.log(weights) + 0.5 * D * np.log(2 * np.pi) + 0.5 * (logdets - logdets.min())
    Q = 0.5 * precs
    Q = 0.5 * (Q + np.transpose(Q, (0, 2, 1)))
    return BodyPrior(means=np.ascontiguousarray(means), Q=np.ascontiguousarray(Q), neglogw=np.ascontiguousarray(neglogw))


def create_gmm_body_prior(pose_body_prior_fname: str, exclude_hands: bool = False) -> BodyPrior:
    gmm = load_reference_pickle(pose_body_prior_fname)
    npose = 63 if exclude_hands else 69
    covars = np.asarray(gmm['covars'], dtype=np.float64)[:, :npose, :npose]
    means = np.asarray(gmm['means'], dtype=np.float64)[:, :npose]
    weights = np.asarray(gmm['weights'], dtype=np.float64).ravel()
    precs = np.stack([np.linalg.inv(c) for c in covars])
    sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in covars])
    const = (2 * np.pi) ** (npose / 2.)
    w = weights / (const * (sqrdets / sqrdets.min()))
    # The reference's residual is sqrt(.5) (x-mu) chol(prec); its square is (x-mu)^T Q (x-mu)
    # with Q = .5 prec, which is all the normal equations need (DESIGN.md "prior term").
    Q = 0.5 * precs
    Q = 0.5 * (Q + np.transpose(Q, (0, 2, 1)))
    return BodyPrior(means=np.ascontiguousarray(means), Q=np.ascontiguousarray(Q),
                     neglogw=np.ascontiguousarray(-np.log(w)))


# --------------------------------------------------------------------------------------
# the device pack
# --------------------------------------------------------------------------------------
@dataclass
class StageIIPack:
    """Constants of one (model, betas, markers_latent) triple, laid out for the device."""
    model_type: str
    n_joints: int
    n_markers: int
    body_dof: int
    p_red: int
    p_full: int
    n_hand_red: int
    n_hand_full: int
    n_dmpl: int              # per-frame linear coefficients in all: DMPL first, then expressions
    kw: int                  # skinning weights kept per slot (ELL width)
    # ---- int arrays
    parents: np.ndarray      # nJ int32
    slot_vid: np.ndarray     # 3M int32 (bookkeeping only)
    w_joint: np.ndarray      # 3M x kw int32 (-1 pad)
    # ---- float64 arrays (converted to the compute type by the library)
    hand_comps: np.ndarray   # n_hand_red x n_hand_full
    hands_mean: np.ndarray   # n_hand_full
    v0: np.ndarray           # 3M x 3    shaped template rows (dmpl = 0)
    sd: np.ndarray           # 3M x 3 x nd
    pd: np.ndarray           # (nJ-1) x 9M x 9   pose-blend slabs, one contiguous slab per joint
    w_val: np.ndarray        # 3M x kw
    j0: np.ndarray           # nJ x 3
    jd: np.ndarray           # nJ x 3 x nd
    coefs: np.ndarray        # M x 3
    # ---- prior
    prior_k: int = 0
    prior_d: int = 0
    prior_off: int = 3
    prior_ids: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))   # non-contiguous prior dimensions (animal models)
    prior_means: np.ndarray = field(default_factory=lambda: np.zeros((0, 0)))
    prior_Q: np.ndarray = field(default_factory=lambda: np.zeros((0, 0, 0)))
    prior_neglogw: np.ndarray = field(default_factory=lambda: np.zeros(0))
    # ---- variable partitions, indices into x = [trans(3) | pose(p_red) | dmpl(nd)]
    free_step1: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    free_step2: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    finger_lo: int = 0       # reduced-pose ids [lo, hi) penalised by poseH in step 2
    finger_hi: int = 0
    face_lo: int = 0         # reduced-pose ids [lo, hi) penalised by poseF in step 2 (the jaw)
    face_hi: int = 0
    n_expr: int = 0          # how many of the n_dmpl linear coefficients (the last ones) are expression coefficients
    jangles_ids: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))    # animal_horse joint-angle term: reduced-pose ids
    jangles_signs: np.ndarray = field(default_factory=lambda: np.zeros(0))            # ... and signs
    # ---- host-only bookkeeping
    closest: np.ndarray = field(default_factory=lambda: np.zeros((0, 3), np.int64))
    can_verts_sel: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))

    @property
    def nx(self) -> int:
        return 3 + self.p_red + self.n_dmpl


def _rodrigues(rv: np.ndarray) -> np.ndarray:
    th = float(np.linalg.norm(rv))
    K = np.array([[0.0, -rv[2], rv[1]], [rv[2], 0.0, -rv[0]], [-rv[1], rv[0], 0.0]])
    if th < 1e-8:
        return np.eye(3) + K
    return np.eye(3) + (np.sin(th) / th) * K + ((1.0 - np.cos(th)) / th ** 2) * (K @ K)


def canonical_verts(model: SurfaceModel, v_shaped: np.ndarray, joints: np.ndarray) -> np.ndarray:
    """The canonical mesh ``can_model.r`` the markers are attached to (chmosh.py:502): the model at
    zero *reduced* pose and zero translation.  That is not the template: with ``use_hands_mean`` the
    full pose of the canonical body carries the mean hand pose (smpl_fast_derivatives.py:194-204).
    One full-mesh LBS evaluation per subject, host side; the per-frame forward is device code."""
    nj = model.n_joints
    full = np.zeros(model.p_full)
    if model.n_joints * 3 > model.body_dof:
        full[model.body_dof:] = model.hands_mean
    if not np.any(full):
        return v_shaped.copy()
    R = np.stack([_rodrigues(full[3 * j:3 * j + 3]) for j in range(nj)])
    posefeat = (R[1:] - np.eye(3)).reshape(-1)
    v_posed = v_shaped + model.posedirs.dot(posefeat)
    Rg = np.zeros((nj, 3, 3))
    tg = np.zeros((nj, 3))
    Rg[0], tg[0] = R[0], joints[0]
    for j in range(1, nj):
        a = model.parents[j]
        Rg[j] = Rg[a] @ R[j]
        tg[j] = tg[a] + Rg[a] @ (joints[j] - joints[a])
    out = np.zeros_like(v_posed)
    for j in range(nj):
        w = model.weights[:, j]
        nz = np.nonzero(w)[0]
        if len(nz):
            out[nz] += w[nz, None] * ((v_posed[nz] - joints[j]) @ Rg[j].T + tg[j])
    return out


def pose_partitions(model_type: str, p_red: int, optimize_fingers: bool, optimize_face: bool,
                    optimize_toes: bool):
    """Reduced-pose id partitions of the reference Stage II (chmosh.py:548-571,645-647,676-692)."""
    all_ids = list(range(p_red))
    root = all_ids[:3]
    body: List[int] = []
    face: List[int] = []
    finger: List[int] = []
    if model_type == 'smpl':
        body = all_ids[3:]
    elif model_type == 'smplh':
        body = all_ids[3:66]
        if optimize_fingers:
            finger = all_ids[66:]
    elif model_type == 'smplx':
        body = all_ids[3:66]
        if optimize_face:
            face = all_ids[66:69]
        if optimize_fingers:
            finger = all_ids[75:]
    elif model_type == 'mano':
        finger = all_ids[3:]
    elif model_type == 'animal_horse':
        body = all_ids[3:84]                                 # tail, mouth and ears stay at rest (chmosh.py:572-573)
    elif model_type == 'animal_dog':
        if p_red < 3 * (DOG_BODY_JOINTS[-1] + 1):
            raise ValueError(f'animal_dog: the pose prior covers joints up to {DOG_BODY_JOINTS[-1]}; this model has '
                             f'{p_red // 3} joints')
        body = [all_ids[i] for i in DOG_BODY_IDS]            # joints 2, 6 and 29 stay at rest (chmosh.py:574-579)
    else:
        # object is listed by the reference but cannot run its Stage II: RigidObjectModel has no `fullpose`
        # (chmosh.py:719); it is not built here
        raise NotImplementedError(f'surface model type {model_type!r} is outside the Stage-II hot path of this build')
    step1 = root + body
    if len(body) and not optimize_toes:
        step1 = sorted(set(step1).difference(all_ids[30:36]))
    step2 = sorted(set(step1 + finger + face))
    return dict(root=root, body=body, face=face, finger=finger, step1=sorted(step1), step2=step2)


def build_pack(model: SurfaceModel, betas: np.ndarray, markers_latent: np.ndarray, *,
               num_betas: int, prior: Optional[BodyPrior], dmpl_dirs: Optional[np.ndarray] = None,
               num_dmpls: int = 0, optimize_fingers: bool = False, optimize_toes: bool = False,
               optimize_face: bool = False, expr_start: int = 0, num_expressions: int = 0,
               can_verts: Optional[np.ndarray] = None, jd_lin: Optional[np.ndarray] = None) -> StageIIPack:
    """``optimize_face`` (SMPL-X, chmosh.py:560-566,685-689): the ``num_expressions`` shape components from
    ``expr_start`` become per-frame linear coefficients after the DMPL ones, and the jaw joins the free pose."""
    nj = model.n_joints
    betas = np.asarray(betas, dtype=np.float64).ravel()
    nb = min(num_betas, model.shapedirs.shape[-1], betas.shape[0])
    v_shaped = model.v_template + model.shapedirs[:, :, :nb].dot(betas[:nb])   # chmosh.py:499-500
    j0 = model.J_regressor.dot(v_shaped)                                       # smpl_fast_derivatives.py:186-191
    if can_verts is None:          # (Stage I hands the canonical mesh in: it keeps it as an affine function of the shape)
        can_verts = canonical_verts(model, v_shaped, j0)                       # can_model.r
    closest, coefs = attach_markers(can_verts, markers_latent)                 # chmosh.py:502
    M = closest.shape[0]
    slot_vid = closest.reshape(-1).astype(np.int64)                            # slot = 3*m + t

    nd = int(num_dmpls) if dmpl_dirs is not None else 0
    if nd:
        dm = np.asarray(dmpl_dirs, dtype=np.float64)[:, :, :nd]
        sd = dm[slot_vid]
        jd = np.einsum('jv,vcd->jcd', model.J_regressor, dm) if jd_lin is None else np.asarray(jd_lin, dtype=np.float64)   # (constant per model)
    else:
        sd = np.zeros((3 * M, 3, 0))
        jd = np.zeros((nj, 3, 0))
    n_expr = 0
    if optimize_face:
        if model.model_type != 'smplx':
            optimize_face = False                                               # chmosh.py:560: only SMPL-X has face ids
        else:
            n_expr = int(num_expressions)
            if expr_start + n_expr > model.shapedirs.shape[-1]:
                raise ValueError(f'the model has {model.shapedirs.shape[-1]} shape components; expressions '
                                 f'{expr_start}..{expr_start + n_expr} do not exist')
            ex = np.asarray(model.shapedirs[:, :, expr_start:expr_start + n_expr], dtype=np.float64)
            sd = np.concatenate([sd, ex[slot_vid]], axis=2)
            jd = np.concatenate([jd, np.einsum('jv,vcd->jcd', model.J_regressor, ex)], axis=2)
    nd_dm, nd = nd, nd + n_expr

    # pose-blend slabs: pd[j-1, 3*slot + c, e] = posedirs[vid(slot), c, 9(j-1)+e]
    pdsel = model.posedirs[slot_vid].reshape(3 * M, 3, nj - 1, 9)
    pd = np.ascontiguousarray(np.transpose(pdsel, (2, 0, 1, 3)).reshape(nj - 1, 9 * M, 9))

    # skinning weights in ELL form
    wsel = model.weights[slot_vid]
    nnz = (wsel != 0).sum(1)
    kw = int(max(1, nnz.max()))
    w_joint = -np.ones((3 * M, kw), dtype=np.int32)
    w_val = np.zeros((3 * M, kw))
    for s in range(3 * M):
        js = np.nonzero(wsel[s])[0]
        w_joint[s, :len(js)] = js
        w_val[s, :len(js)] = wsel[s, js]
    if kw > 8:
        raise ValueError(f'a marker vertex has {kw} non-zero skinning weights; the kernel keeps at most 8 per vertex')

    parts = pose_partitions(model.model_type, model.p_red, optimize_fingers, optimize_face, optimize_toes)
    p_red = model.p_red
    step1 = [0, 1, 2] + [3 + i for i in parts['step1']]
    step2 = [0, 1, 2] + [3 + i for i in parts['step2']] + [3 + p_red + i for i in range(nd)]
    finger = parts['finger']
    f_lo, f_hi = (finger[0], finger[-1] + 1) if finger else (0, 0)
    assert not finger or finger == list(range(f_lo, f_hi))
    face = parts['face']
    c_lo, c_hi = (face[0], face[-1] + 1) if face else (0, 0)
    assert not face or face == list(range(c_lo, c_hi))

    pack = StageIIPack(
        model_type=model.model_type, n_joints=nj, n_markers=M, body_dof=model.body_dof, p_red=p_red,
        p_full=model.p_full, n_hand_red=model.hand_comps.shape[0], n_hand_full=model.hands_mean.shape[0],
        n_dmpl=nd, n_expr=n_expr, kw=kw,
        parents=model.parents.astype(np.int32),
        slot_vid=slot_vid.astype(np.int32), w_joint=w_joint,
        hand_comps=np.ascontiguousarray(model.hand_comps), hands_mean=np.ascontiguousarray(model.hands_mean),
        v0=np.ascontiguousarray(v_shaped[slot_vid]), sd=np.ascontiguousarray(sd), pd=pd,
        w_val=np.ascontiguousarray(w_val), j0=np.ascontiguousarray(j0), jd=np.ascontiguousarray(jd),
        coefs=coefs,
        free_step1=np.asarray(step1, dtype=np.int32), free_step2=np.asarray(step2, dtype=np.int32),
        finger_lo=int(f_lo), finger_hi=int(f_hi), face_lo=int(c_lo), face_hi=int(c_hi),
        closest=closest, can_verts_sel=np.ascontiguousarray(can_verts[slot_vid]),
    )
    if len(parts['body']):
        if prior is None:
            raise KeyError("pose")  # the reference indexes opt_model.priors['pose'] (chmosh.py:614)
        d = len(parts['body'])
        if prior.means.shape[1] != d:
            raise ValueError(f'body prior has {prior.means.shape[1]} dims, pose body has {d}')
        pack.prior_k = prior.means.shape[0]
        pack.prior_d = d
        pack.prior_off = parts['body'][0]
        if parts['body'] != list(range(pack.prior_off, pack.prior_off + d)):     # (the dog: joints with gaps)
            pack.prior_ids = np.asarray(parts['body'], dtype=np.int32)
        pack.prior_means = prior.means
        pack.prior_Q = prior.Q
        pack.prior_neglogw = prior.neglogw
    if model.model_type == 'animal_horse':
        pack.jangles_ids, pack.jangles_signs = HORSE_JANGLES_IDS.copy(), HORSE_JANGLES_SIGNS.copy()
    return pack
