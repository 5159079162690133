"""The normal equations of one frame (mosh2_job_linearize), in float64 and float32, against the float64 oracle at the state
the kernel was given.

The parity and same-state tests see the linearisation only through converged solutions, and the dog-leg hides a wrong
Jacobian there: rho is computed from the true SSE, so a slightly wrong A or g changes the path to the minimum, not the
minimum.  Here every output of one linearisation is compared on its own: the weighted data rows J (3M x n), the residual r,
the posed attachment vertices, the simulated markers, A = J^T J of all the frame's terms, g = -J^T r and the SSE columns.

Inputs.  Every family of conftest.SMALL, Step 1 and Step 2 (the hand tile runs only where finger columns are free: Step 2 of
C2, C3, C4 and CF), at the first frames of a float64 solve and at the same states perturbed by N(0, 0.05) rad / 5 mm, with
three markers of one frame hidden.  C2 repeats with the finger term switched off.  The reference is
``oracle.stageii._Objective`` with linearise mode's terms -- data at wt_data (no marker-count scaling, no visibility
annealing), the pose prior (+ the horse's joint angles), in Step 2 the finger, jaw / expression and (C3, optimize_dynamics)
DMPL terms -- evaluated at the state the kernel held: in float32 the rounded state and the rounded observations.  Max-mixture: the kernel picks the
component in its own precision, so the reference uses the component whose float64 energy, within ``margin`` of the minimum,
gives the kernel's poseB SSE.

Measures (per frame, maxima over frames):
  J     |J - J_ref| / max |J_ref[:, col]| per column; rows of hidden markers exactly zero
  r     |r - r_ref| / wt_data (metres), vp / markers |. - ref| (metres)
  A     |A_ij - A_ref_ij| / sqrt(A_ref_ii A_ref_jj)
  g     |g - g_ref| / (sqrt(A_ref_ii) |r_all|), r_all the residual of all terms
  SSE   relative to the float64 value; the data SSE relative to 2 |r_data| (wt_data sqrt(3 n_vis)) (its residual cancels)
Float64 bounds: summation order only.  Float32 bounds: 4x the maxima of the single-thread host build of the same source in
float32 over the same inputs (the CPU twin below), per family; ``TWIN_F32`` lists those maxima.  The largest, J 1.4e-4 of
the column's largest entry, is on CF's hand-pose columns.  The GPU's J^T J runs on the tensor cores in split TF32
(tests/tc/jtj_tf32_test.cu: 1.5e-6 of the largest diagonal), so where it does its A may in addition be off by
1.5e-6 max_i A_ii.  That allowance is absolute: on the columns with the smallest diagonals (the finger and expression
coefficients, whose A_ii are orders of magnitude below the translation's) it is looser than the relative bound, and a
defect confined to those columns' data part would have to exceed it.  The tensor cores build A for float32 jobs except
in the global-workspace layout and under MOSH2_DEV_NO_TC=1 (``carve``'s ``tc_ok``); every family's float32 workspace fits
shared memory, so no default launch falls back to the global workspace.

The DMPL term: the kernel's closed-form terms add wt_dmpl^2 to the DMPL coefficients' diagonal in Step 2 whenever the job's
options have optimize_dynamics, linearise mode included, so the reference has it too (C3).
"""
import copy
import ctypes as C

import numpy as np
import pytest

from conftest import dense_obs, gpu_solve
from moshpp_b200 import lib

COL = {k: i for i, k in enumerate(lib.ERR_NAMES)}
PREC = {'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}
TC_A = 1.5e-6            # split-TF32 J^T J, of the largest diagonal entry

# float32: the CPU twin's maxima per family over Step 1, Step 2 and (C2) the finger term off; the bounds are 4x these
TWIN_F32 = {
    'C1': dict(J=2.6e-6, r=1.8e-7, vp=2.2e-7, markers=1.8e-7, A=2.1e-6, g=3.1e-6, sse=2.5e-7, data=8.7e-9),
    'C2': dict(J=2.2e-5, r=6.9e-7, vp=2.7e-7, markers=6.9e-7, A=8.0e-6, g=1.1e-5, sse=2.9e-7, data=8.0e-9),
    'C3': dict(J=7.6e-5, r=4.2e-7, vp=3.4e-7, markers=4.5e-7, A=1.9e-5, g=1.4e-5, sse=2.7e-7, data=1.2e-8),
    'C4': dict(J=6.6e-7, r=9.5e-8, vp=3.6e-8, markers=9.5e-8, A=7.2e-7, g=5.8e-6, sse=1.0e-7, data=5.2e-9),
    'CF': dict(J=1.4e-4, r=7.2e-7, vp=3.5e-7, markers=7.2e-7, A=6.9e-5, g=9.4e-6, sse=4.0e-7, data=1.1e-8),
    'CH': dict(J=2.6e-6, r=5.9e-7, vp=4.1e-7, markers=5.9e-7, A=2.3e-6, g=1.4e-5, sse=2.3e-7, data=2.5e-8),
}
F64 = dict(J=1e-10, r=1e-12, vp=1e-12, markers=1e-12, A=1e-10, g=1e-10, sse=1e-10, data=1e-12)
MARGIN = {'f64': 0.0, 'f32': 4.6e-6}     # the max-mixture margin of tests/test_gpu_same_state.py
FAMILIES = list(TWIN_F32)


def tolerance(name, precision):
    return F64 if precision == 'f64' else {k: 4 * v for k, v in TWIN_F32[name].items()}


N_STATES = 3             # solved frames per case; each also perturbed -> 2 N_STATES linearised frames


def _solver(case):
    from oracle import stageii
    return stageii.StageIISolver(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def _prepare(case, fingers=True):
    from moshpp_b200 import chmosh
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    if not fingers:
        opts.optimize_fingers = 0
    return pk, opts


def lin_inputs(case, res):
    """States and observations of the linearised frames: the first N_STATES solved frames of ``res`` as they are, then the
    same perturbed; markers 0, 5 and M-1 of the second frame hidden."""
    obs, vis = dense_obs(case)
    pk = case['pack']
    solved = np.nonzero(res.status & lib.ST_SOLVED)[0][:N_STATES]
    assert len(solved) == N_STATES
    x = np.concatenate([res.trans[solved], res.pose[solved], res.dmpls[solved, :pk.n_dmpl]], axis=1)
    rng = np.random.default_rng(7)
    xp = x + np.concatenate([rng.normal(0, 0.005, (N_STATES, 3)), rng.normal(0, 0.05, (N_STATES, x.shape[1] - 3))], axis=1)
    o = np.concatenate([obs[solved], obs[solved]])
    v = np.concatenate([vis[solved], vis[solved]]).astype(np.uint8)
    for i in (0, 5, pk.n_markers - 1):
        v[1, i] = 0
        o[1, i] = 0.0
    return np.ascontiguousarray(o), np.ascontiguousarray(v), np.ascontiguousarray(np.concatenate([x, xp]))


def reference(solver, opts, step, obs, vis, x, poseB_sse, margin):
    """The float64 oracle of one linearised frame at state ``x`` (observations ``obs`` M x 3, visibility ``vis``).  With a
    max-mixture prior the component is the one (within ``margin`` of the float64 minimum) whose energy matches the
    kernel's ``poseB_sse``."""
    from oracle import stageii
    s = solver
    PR = len(s.pose)
    s.trans[:] = x[:3]
    s.pose[:] = x[3:3 + PR]
    if s.nd:
        s.betas[s.lin_ids] = x[3 + PR:]
    terms = [['data', opts.wt_data]]
    prior = s.prior
    if len(s.body_ids):
        terms.append(['poseB', opts.wt_poseB])
        if s.model.model_type == 'animal_horse':
            terms.append(['poseB_jangles', 2.0 * opts.wt_poseB])
        if hasattr(prior, 'weights'):
            xb = s.pose[s.body_ids]
            en = np.array([(l ** 2).sum() - np.log(w) for l, w in zip(prior.loglikelihoods(xb), prior.weights)])
            cand = np.nonzero(en <= en.min() + margin * max(1.0, abs(en.min())))[0]
            k = int(cand[np.argmin(np.abs(opts.wt_poseB ** 2 * en[cand] - poseB_sse))])
            fixed = copy.copy(prior)
            fixed.select = lambda xx, k=k: (k, fixed.loglikelihoods(xx)[k])
            s.prior = fixed
    if step == 2:
        if opts.optimize_fingers and len(s.finger_ids):
            terms.append(['poseH', opts.wt_poseH])
        if opts.optimize_face and len(s.face_ids):
            terms.append(['poseF', opts.wt_poseF])
            terms.append(['expr', opts.wt_expr])
        if opts.optimize_dynamics:
            terms.append(['dmpl', opts.wt_dmpl])
    vidx = np.nonzero(vis)[0]
    ids = s.step2_ids if step == 2 else s.step1_ids
    obj = stageii._Objective(s, obs[vidx], vidx, terms, ids, step == 2 and s.nd > 0)
    try:
        r_all, J_all = obj(obj.x0(), True)
        sse = obj.term_sse()
    finally:
        s.prior = prior
    M, n, nv = s.n_markers, obj.n, len(vidx)
    rows = (3 * vidx[:, None] + np.arange(3)).ravel()
    J = np.zeros((3 * M, n))
    J[rows] = J_all[:3 * nv]
    r = np.zeros(3 * M)
    r[rows] = r_all[:3 * nv]
    verts = s.lbs(s.pose, s.betas, s.trans, False, beta_ids=s.lin_ids)
    vp = verts[s.tri.reshape(-1)]
    return dict(J=J, r=r, vp=vp, markers=s.evaluate(False)['markers'], A=J_all.T @ J_all, g=-J_all.T @ r_all,
                r_all=r_all, sse=sse, n_vis=nv, terms=dict(terms))


def normal_equation_errors(case, name, pk, opts, step, obs, vis, x, out, precision, tc=False):
    """Compares the linearisation ``out`` (mosh2_lin_out arrays, build = 1) of family ``name`` with the oracle frame by
    frame and asserts the bounds of ``tolerance``; ``tc``: A from the split-TF32 J^T J.  Returns the maxima per measure."""
    tol = tolerance(name, precision)
    solver = _solver(case)
    n = len(pk.free_step2 if step == 2 else pk.free_step1)
    assert n == 3 + len(solver.step2_ids if step == 2 else solver.step1_ids) + (solver.nd if step == 2 else 0)
    col = dict(COL, poseB_jangles=COL['poseH']) if solver.model.model_type == 'animal_horse' else COL
    if precision == 'f32':             # the state and the observations the kernel held
        obs, x = obs.astype(np.float32).astype(np.float64), x.astype(np.float32).astype(np.float64)
    st = {k: 0.0 for k in ('J', 'r', 'vp', 'markers', 'A', 'g', 'sse', 'data')}
    for f in range(x.shape[0]):
        ref = reference(solver, opts, step, obs[f], vis[f], x[f], out['errs'][f, COL['poseB']], MARGIN[precision])
        hidden = np.repeat(vis[f] == 0, 3)
        assert not np.any(out['J'][f][hidden]) and not np.any(out['r'][f][hidden]), f
        e = {}
        e['J'] = (np.abs(out['J'][f] - ref['J']) / np.maximum(np.abs(ref['J']).max(0), 1e-300)).max()
        e['r'] = np.abs(out['r'][f] - ref['r']).max() / opts.wt_data
        e['vp'] = np.abs(out['vp'][f] - ref['vp']).max()
        e['markers'] = np.abs(out['markers_sim'][f] - ref['markers']).max()
        d = np.sqrt(np.diag(ref['A']))
        dA = np.abs(out['A'][f] - ref['A'])
        if tc:
            dA = np.maximum(dA - TC_A * d.max() ** 2, 0.0)
        e['A'] = (dA / np.outer(d, d)).max()
        e['g'] = (np.abs(out['g'][f] - ref['g']) / (d * np.linalg.norm(ref['r_all']))).max()
        e['sse'] = 0.0
        for c, k in enumerate(lib.ERR_NAMES):              # columns of the terms linearise mode does not have stay zero
            if not any(col[term] == c for term in ref['sse']):
                assert out['errs'][f, c] == 0.0, (f, k)
        for term, v in ref['sse'].items():
            got = out['errs'][f, col[term]]
            if term == 'data':
                wt, n3 = ref['terms']['data'], 3 * ref['n_vis']
                e['data'] = abs(got - v) / (2 * np.sqrt(v) * wt * np.sqrt(n3))
            else:
                e['sse'] = max(e['sse'], abs(got - v) / max(abs(v), 1e-300))
        for k, v in e.items():
            assert v <= tol[k], (f, k, v, tol[k])
            st[k] = max(st[k], float(v))
    return st


# ---- CPU twin: the single-thread host build of the device source, both precisions --------------------------------------

@pytest.fixture(scope='module')
def emu_lin():
    from moshpp_b200 import build
    handle = C.CDLL(build.build_emu())

    def run(pk, opts, obs, vis, x, step, precision):
        F, M = obs.shape[0], pk.n_markers
        n = len(pk.free_step2 if step == 2 else pk.free_step1)
        h = lib.DescHolder(pk)
        out = dict(errs=np.zeros((F, len(lib.ERR_NAMES))), markers_sim=np.zeros((F, M, 3)), r=np.zeros((F, 3 * M)),
                   vp=np.zeros((F, 3 * M, 3)), A=np.zeros((F, n, n)), g=np.zeros((F, n)), J=np.zeros((F, 3 * M, n)))
        c = lib.LinOut(*[lib._ptr(out[k], lib._f64p) for k in ('errs', 'markers_sim', 'r', 'vp', 'A', 'g', 'J')])
        rc = handle.mosh2_emu_linearize_precision(C.byref(h.desc), C.byref(opts), F, lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p),
                                                  int(step), 1, lib._ptr(x, lib._f64p), PREC[precision], C.byref(c))
        assert rc == 0
        return out
    return run


@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', FAMILIES + ['C2-nofingers'])
def test_device_source_normal_equations_equal_float64(cases, emu, emu_lin, name, step, precision):
    case = cases(name.split('-')[0])
    pk, opts = _prepare(case, fingers=not name.endswith('nofingers'))
    obs, vis, x = lin_inputs(case, emu(case))
    out = emu_lin(pk, opts, obs, vis, x, step, precision)
    st = normal_equation_errors(case, name.split('-')[0], pk, opts, step, obs, vis, x, out, precision)
    print(name, step, precision, {k: float('%.2g' % v) for k, v in st.items()})


# ---- the CUDA kernel -------------------------------------------------------------------------------------------------

def gpu_linearize(pk, opts, obs, vis, x, step, precision):
    model = lib.Model(pk, device=0)
    try:
        job = model.job(obs.shape[0], opts, chunk_len=1, chunk_warmup=0, precision=PREC[precision])
        try:
            job.upload(obs, vis)
            return job.linearize(x, opts, step, True)
        finally:
            job.close()
    finally:
        model.close()


@pytest.fixture(scope='module')
def gpu_states():
    cache = {}

    def get(case, name):
        if name not in cache:
            cache[name] = lin_inputs(case, gpu_solve(case, precision='f64'))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', FAMILIES + ['C2-nofingers'])
def test_kernel_normal_equations_equal_float64(cases, gpu_states, name, step, precision):
    case = cases(name.split('-')[0])
    pk, opts = _prepare(case, fingers=not name.endswith('nofingers'))
    obs, vis, x = gpu_states(case, name.split('-')[0])
    out = gpu_linearize(pk, opts, obs, vis, x, step, precision)
    st = normal_equation_errors(case, name.split('-')[0], pk, opts, step, obs, vis, x, out, precision, tc=precision == 'f32')
    print(name, step, precision, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.gpu
def test_kernel_linearize_takes_the_face_weights_of_the_call(cases, gpu_states, emu_lin):
    """mosh2_job_linearize evaluates the jaw and expression terms under the call's wt_poseF and wt_expr (Stage I anneals its
    weights between minimisations), not under those the job was created with: a float64 job created with CF's options and
    linearised with both weights tripled equals the host build given the tripled weights."""
    case = cases('CF')
    pk, opts = _prepare(case)
    obs, vis, x = gpu_states(case, 'CF')
    call = lib.Options.from_buffer_copy(opts)
    call.wt_poseF *= 3
    call.wt_expr *= 3
    model = lib.Model(pk, device=0)
    try:
        job = model.job(obs.shape[0], opts, chunk_len=1, chunk_warmup=0, precision=lib.MOSH2_F64)
        try:
            job.upload(obs, vis)
            got = job.linearize(x, call, 2, True)['errs']
        finally:
            job.close()
    finally:
        model.close()
    want = emu_lin(pk, call, obs, vis, x, 2, 'f64')['errs']
    for term in ('poseF', 'expr'):
        ref = want[:, COL[term]]
        assert np.all(ref > 0), term
        assert np.abs(got[:, COL[term]] - ref).max() <= F64['sse'] * ref.max(), term


@pytest.mark.gpu
@pytest.mark.parametrize('switch', [('MOSH2_DEV_NO_TC', '1'), ('MOSH2_DEV_TILE', '10'), ('MOSH2_DEV_BIG', '1'),
                                    ('MOSH2_DEV_THREADS', '256'), ('MOSH2_DEV_THREADS', '128')])
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', ['C2', 'CF'])
def test_f32_kernel_normal_equations_under_other_launch_layouts(cases, gpu_states, name, step, switch, monkeypatch):
    """The float32 linearisation with the register-tile J^T J, 10-marker tiles, A and the Jacobian tiles in a global
    workspace, and 256 or 128 threads instead of 384; the same bounds.  The tile, workspace and tensor-core switches are read
    when the job is created, the thread count at every launch."""
    case = cases(name)
    pk, opts = _prepare(case)
    obs, vis, x = gpu_states(case, name)
    monkeypatch.setenv(*switch)
    out = gpu_linearize(pk, opts, obs, vis, x, step, 'f32')
    monkeypatch.delenv(switch[0])
    tc = switch[0] not in ('MOSH2_DEV_NO_TC', 'MOSH2_DEV_BIG')     # the layouts whose J^T J runs on the tensor cores
    st = normal_equation_errors(case, name, pk, opts, step, obs, vis, x, out, 'f32', tc=tc)
    print(name, step, switch, {k: float('%.2g' % v) for k, v in st.items()})
