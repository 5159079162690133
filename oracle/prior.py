"""Body-pose priors (oracle; test infrastructure only).

Reference: prior/gmm_prior_ch.py:42-85 (MaxMixtureComplete) and :107-134 (create_gmm_body_prior), prior/dog_body_prior.py:53-87
(the dog's max-mixture), prior/horse_body_prior.py:40-71 (the horse's Gaussian and joint-angle terms).
"""
from __future__ import annotations

import pickle

import numpy as np


class MaxMixtureComplete:
    def __init__(self, means, precs, weights):
        self.means = np.asarray(means, dtype=np.float64)
        self.precs = np.asarray(precs, dtype=np.float64)     # chol(inv(cov)), lower (line 123)
        self.weights = np.asarray(weights, dtype=np.float64).ravel()

    def loglikelihoods(self, x):
        return [np.sqrt(0.5) * (x - m).dot(s) for m, s in zip(self.means, self.precs)]   # line 56

    def select(self, x):
        ll = self.loglikelihoods(x)
        k = int(np.argmin([(l ** 2).sum() - np.log(w) for l, w in zip(ll, self.weights)]))   # lines 59-62
        return k, ll[k]

    def r(self, x):
        k, l = self.select(x)
        return np.concatenate((l, [np.sqrt(-np.log(self.weights[k]))]))                     # lines 69-72

    def dr_wrt_x(self, x):
        """(D+1) x D with an empty last row (lines 74-85)."""
        k, _ = self.select(x)
        d = len(x)
        J = np.zeros((d + 1, d))
        J[:d] = np.sqrt(0.5) * self.precs[k].T
        return J


def create_gmm_body_prior(pose_body_prior_fname, exclude_hands=False) -> MaxMixtureComplete:
    with open(pose_body_prior_fname, 'rb') as f:
        gmm = pickle.load(f, encoding='latin-1')
    npose = 63 if exclude_hands else 69
    covars = gmm['covars'][:, :npose, :npose]
    means = gmm['means'][:, :npose]
    weights = gmm['weights']
    precs = np.asarray([np.linalg.inv(cov) for cov in covars])
    chols = np.asarray([np.linalg.cholesky(prec) for prec in precs])
    sqrdets = np.array([(np.sqrt(np.linalg.det(c))) for c in covars])
    const = (2 * np.pi) ** (npose / 2.)
    weights = weights / (const * (sqrdets / sqrdets.min()))
    return MaxMixtureComplete(means=means, precs=chols, weights=weights)


# the dog's body pose ids (chmosh.py:304-309,574-579): joints 1, 3-5, 7-28 and 30-34 of its 35, i.e. 93 ids with gaps
DOG_JOINTS = [1, 3, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 30, 31, 32, 33, 34]
DOG_POSE_IDS = np.arange(0, 105).reshape([-1, 3])[DOG_JOINTS].reshape(-1)


def dog_oracle_prior(prior_pklpath) -> MaxMixtureComplete:
    """MaxMixtureDog.get_gmm_prior (prior/dog_body_prior.py:53-87), with the check its message describes: the reference asserts
    that some determinant IS zero (lines 78-79), while the message and the division on line 83 mean the opposite."""
    with open(prior_pklpath, 'rb') as f:
        gmm = pickle.load(f, encoding='latin-1')
    npose = len(DOG_POSE_IDS)
    covars = gmm['gmm_covs'][:, :, DOG_POSE_IDS][:, DOG_POSE_IDS]
    means = gmm['gmm_means'][:, DOG_POSE_IDS]
    weights = gmm['gmm_weights'][:]
    precs = np.asarray([np.linalg.inv(cov) for cov in covars])
    chols = np.asarray([np.linalg.cholesky(prec) for prec in precs])
    sqrdets = np.array([(np.sqrt(np.linalg.det(c))) for c in covars])
    if np.any(sqrdets == 0.0):
        raise ValueError(f'Encountered zeros in the determinant of the covariance matrix:  {sqrdets}')
    const = (2 * np.pi) ** (npose / 2.)
    weights = weights / (const * (sqrdets / sqrdets.min()))
    return MaxMixtureComplete(means=means, precs=chols, weights=weights)


def create_body_prior(model_type, pose_body_prior_fname):
    """The body pose prior of a model type (bodymodel_loader.py:121-131): None without a file and for MANO."""
    if not pose_body_prior_fname or model_type == 'mano':
        return None
    if model_type == 'animal_horse':
        return HorsePosePrior(pose_body_prior_fname)
    if model_type == 'animal_dog':
        return dog_oracle_prior(pose_body_prior_fname)
    return create_gmm_body_prior(pose_body_prior_fname, exclude_hands=model_type in ('smplh', 'smplx'))


class HorsePosePrior:
    """smal_horse_prior (prior/horse_body_prior.py:40-53, disable_tail_mouth_ear): r(x) = (x - mean_pose[:81]) . pic[:81, :81]."""

    def __init__(self, prior_pklpath):
        with open(prior_pklpath, 'rb') as f:
            res = pickle.load(f, encoding='latin-1')
        self.precs = np.asarray(res['pic'], dtype=np.float64)[:81, :81]
        self.means = np.asarray(res['mean_pose'], dtype=np.float64)[:81]

    def r(self, x):
        return (x - self.means).dot(self.precs)

    def dr_wrt_x(self, x):
        return self.precs.T


# smal_horse_joint_angle_prior (prior/horse_body_prior.py:56-71): entries of pose[3:84], i.e. pose ids 6, 7, 8, ... ; signs +1
HORSE_JANGLES_IDS = np.array([6, 7, 8, 11, 12, 13, 20, 21, 22, 25, 26, 27]) - 3
HORSE_JANGLES_SIGNS = np.ones(12)


def horse_joint_angles(body_pose):
    """power(exp(pose[idx] * sign), 2)"""
    return np.exp(body_pose[HORSE_JANGLES_IDS] * HORSE_JANGLES_SIGNS) ** 2
