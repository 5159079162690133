"""Builds oracle/_ref/: the parts of the reference that compile here from their own sources (test infrastructure).

  libs2m.so   scan2mesh/mesh_distance/sample2meshdist.h + robust.h, UNMODIFIED and compiled where they lie under
              /root/reference, behind the C wrappers of oracle/s2m_wrap.cpp.  The header needs Eigen only as a
              3-vector / 3x3 container; Eigen is not installed, so it compiles against the stand-in oracle/eigen_shim.
              (The reference's own build -- Cython + CGAL for the AABB tree of psbody.mesh -- is not runnable here.)

    python -m oracle.build_ref            # needs the reference sources
tests/golden/make_reference_vectors.py stores what the header computes (ref_s2m.npz); the tests read only that.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = '/root/reference/src/moshpp/scan2mesh/mesh_distance'
OUT = os.path.join(HERE, '_ref', 'libs2m.so')


def build(force: bool = False) -> str:
    """Returns the path of libs2m.so, building it when the reference sources are present; '' if neither exists."""
    if os.path.exists(os.path.join(REF_DIR, 'sample2meshdist.h')):
        srcs = [os.path.join(HERE, 's2m_wrap.cpp'), os.path.join(REF_DIR, 'sample2meshdist.h'), os.path.join(REF_DIR, 'robust.h'),
                os.path.join(HERE, 'eigen_shim', 'eigen3', 'Eigen', 'Core')]
        stale = not os.path.exists(OUT) or any(os.path.getmtime(s) > os.path.getmtime(OUT) for s in srcs)
        if force or stale:
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            cmd = ['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-w', '-I', REF_DIR, '-I', os.path.join(HERE, 'eigen_shim'),
                   '-o', OUT, srcs[0]]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError('g++ failed:\n' + r.stdout + r.stderr)
    return OUT if os.path.exists(OUT) else ''


if __name__ == '__main__':
    print(build(force=True) or 'reference sources not found and no prebuilt library')
