"""mosh2-b200: an H100-native MoSh++ Stage-II pose solver.

The package holds only what the Stage-II hot path needs (SURVEY.md section 8):

* ``chmosh.mosh_stageii``  -- drop-in for the reference's Stage-II callable
  (reference: src/moshpp/chmosh.py:458-741), running on ``libmosh2.so``.
* ``lib``                  -- ctypes binding of the C-ABI in ``include/mosh2.h``.
* ``pack``                 -- once-per-sequence host preprocessing (marker attachment,
  selected-vertex packing) that feeds the device solver.
* ``mocap_interface``      -- mocap readers (npz/pkl/c3d) with the reference's visibility rule.
* ``synth``                -- procedural body models / layouts / motions for tests and bench.
* ``shard``                -- sequence sharding over the GPUs of one box.
* ``mosh_head``            -- MoSh++ end to end without the reference (``MoSh``, ``run_moshpp_once``,
  ``run_moshpp_subject``: a subject's captures in one launch via ``chmosh.mosh_stageii_batch``),
  on ``cfg.prepare_cfg`` and ``frame_picker``.

There is no CPU solver in this package: every solve goes through the CUDA library and
fails loudly when it is missing.
"""

__version__ = "0.1.0"
