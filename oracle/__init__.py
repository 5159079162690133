"""CPU float64 restatement of MoSh++ Stage I and Stage II -- TEST INFRASTRUCTURE ONLY.

One solver per stage (``stagei.StageISolver`` / ``stagei.mosh_stagei``, ``stageii.StageIISolver`` / ``stageii.mosh_stageii``),
with the product's options as keywords: Stage I's ``face_with_free_shape``, ``reference_options`` and ``robust_data_sigma``,
Stage II's ``robust_data_sigma``; ``moshpp.optimize_face`` in cfg in both stages; every body family of the product, the dog
included, as a model type.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import this package; the product (``moshpp_b200``) never does.

PARITY: PINNED TO THE REFERENCE'S OWN CODE wherever that code runs in the build container, UNPINNED for the two external
packages it calls.  The reference (nghorbani/moshpp @ 6599a2d) ships no tests, golden vectors or fixtures for this path
(SURVEY.md section 4).  Pinned, each by vectors / a binary produced from the UNMODIFIED reference files (generators
tests/golden/make_reference_vectors.py and oracle/build_ref.py; tests tests/test_reference_vectors.py,
tests/test_mesh_distance.py):

  * ``rigid.py``          <- moshpp/rigid_transformations.py (imports here as is)                    tests/golden/ref_rigid.npz
  * ``prior.py``          <- moshpp/prior/gmm_prior_ch.py  }  import against a forward-only chumpy   tests/golden/ref_prior.npz
  * ``markers.py``        <- moshpp/transformed_lm.py      }  stand-in (tests/golden/ref_shim)       tests/golden/ref_lms.npz
  * ``mesh_distance.py``  <- scan2mesh/mesh_distance/sample2meshdist.h + robust.h, compiled where they lie against an Eigen
                             stand-in (oracle/eigen_shim) into oracle/_ref/libs2m.so
  * ``robust.py``         <- scan2mesh/robustifiers.py (GMOf)                                         tests/golden/ref_gmof.npz

UNPINNED -- third-party modules that are neither vendored nor installable here, restated from their published algorithms:

  * ``chumpy`` (requirements.txt:2, unpinned; PyPI latest 0.70) -- ``ch.minimize(method='dogleg')``
    call sites chmosh.py:651-653,669-671,703-705.  Restated in ``dogleg.py`` from the published
    algorithm (chumpy/optimization_internal.py ``_minimize_dogleg`` / ``DoglegState``).
  * ``psbody.smpl`` (MPI-internal, never published) -- ``verts_decorated`` and the C++
    ``lbs_derivatives_wrt_pose/_shape`` called at models/smpl_fast_derivatives.py:206-218,246-263.
    Restated in ``lbs.py`` from the public SMPL formulation (``lrotmin`` pose features, LBS).
  * the frame loop itself (``stageii.py`` <- chmosh.py:458-741) and Stage I (``stagei.py`` <- chmosh.py:83-455) cannot run
    without those two and are restatements.

What checks the unpinned parts (SURVEY.md 8(c)): analytic Jacobians == torch.autograd Jacobians of an
independently written float64 forward; cv2.Rodrigues value + Jacobian; scipy least_squares optimum
cross-check; ground-truth recovery on noise-free synthetic data; committed golden vectors emitted
by this oracle (tests/golden/, generator scripts tests/golden/make_golden.py, make_long_golden.py).

Every function cites the reference file:line it follows (paths relative to
/root/reference/src/moshpp unless noted).
"""
