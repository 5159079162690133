"""Development tool (GPU): solve one small case once.  Usage: python tools/gpu_one.py C4 f32"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import conftest  # noqa: E402
from moshpp_b200 import synth  # noqa: E402

name, prec = sys.argv[1], sys.argv[2]
case = synth.make_case(tempfile.mkdtemp(), name, **conftest.SMALL[name])
r = conftest.gpu_solve(case, precision=prec)
print(name, prec, 'builds', r.counters[:, 2].tolist(), 'status', r.status.tolist(), 'pose[1][:4]', r.pose[1][:4])
