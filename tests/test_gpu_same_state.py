"""The Stage-II kernels' output, re-evaluated in float64 at the state they report; and the boundary check's reduction kernel.

Every emitted frame reports a state (pose, trans, dmpls) and, from the kernel's own evaluation AT that state, fullpose,
markers_sim (all M markers, seen or not) and the eight per-term SSEs.  The float64 oracle rebuilds the frame's Step-2
objective (``StageIISolver.frame_terms``) with the targets taken from the kernel's own rows and evaluates it at the
reported state.  The parity tests compare converged solutions, and a least-squares fit moves the pose until a forward
pass that is slightly off fits the observations again; here such an error shows up as itself.

Velocity target: 2 pose[f1] - pose[f2], f1 and f2 the two previous solved frames of the same trajectory; DMPL target:
dmpls[f1] (SURVEY.md Appendix B-1, oracle/stageii.py).  Frames whose predecessors are warm-up frames that were never
emitted skip only the ``velo`` and ``extrap_dmpl`` columns.  The horse's joint-angle SSE is reported in the ``poseH``
column.  The max-mixture prior: the kernel picks the arg-min component in its own precision, so its ``poseB`` SSE is
accepted when it is the SSE of a component whose float64 energy is within ``margin`` of the minimum (zero in float64).

Float32 bounds.  Calibrated on the single-thread host build of the same source in float32 (the CPU twin below: every
family at the sizes of conftest.SMALL); the maxima over all frames were
    fullpose 1.3e-7, markers 6.8e-7 m,
    SSE relative to the float64 value: poseB 5.7e-7, velo 2.3e-7, poseH 2.7e-7, dmpl 1.6e-7, extrap_dmpl 8.6e-8,
    poseF 2.5e-7, expr 8.3e-8.
The bounds are 4x those maxima.  The data SSE is not held to a relative bound: with r = m - obs the residual cancels, so
its bound follows from the marker bound delta (plus the float32 rounding of the observations, 2^-24 |obs|):
    |dSSE| <= wt^2 (2 |r| sqrt(3n) delta + 3n delta^2) + (3n + 8) 2^-24 SSE
over the n visible markers (the last term: the rounding of the weight and of the sum itself).
"""
import numpy as np
import pytest

from conftest import dense_obs, gpu_solve
from moshpp_b200 import lib

EPS32 = 2.0 ** -24
COL = {k: i for i, k in enumerate(lib.ERR_NAMES)}

# float64: summation order only.  float32: 4x the CPU twin's maxima (module docstring); the mixture margin is twice the
# poseB bound (either of two component energies may be off by it).
TOL = {
    'f64': dict(fullpose=1e-12, markers=1e-12, rel=dict.fromkeys(lib.ERR_NAMES, 1e-10), margin=0.0),
    'f32': dict(fullpose=5.2e-7, markers=2.7e-6, margin=4.6e-6,
                rel=dict(poseB=2.3e-6, velo=9.2e-7, poseH=1.1e-6, dmpl=6.4e-7, extrap_dmpl=3.4e-7, poseF=1.0e-6, expr=3.3e-7)),
}


def _solver(case):
    from oracle import stageii
    return stageii.StageIISolver(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def same_state_errors(case, res, precision, seg_start=None, obs_vis=None):
    """Re-evaluates every solved frame of ``res`` in float64 at its reported state and asserts the bounds of ``TOL``.
    ``seg_start[f]``: first emitted frame of the trajectory frame f continues (0 for the sequential pass; the chunk's first
    frame for a chunk with its own warm-up).  Returns the maxima per quantity (errors of the SSEs relative to their value,
    of the data SSE relative to its bound)."""
    from oracle import stageii
    tol = TOL[precision]
    pk = case['pack']
    solver = _solver(case)
    obs, vis = obs_vis if obs_vis is not None else dense_obs(case)
    F = obs.shape[0]
    seq = seg_start is None
    seg = np.zeros(F, dtype=np.int64) if seq else np.asarray(seg_start)
    solved = np.nonzero(res.status & lib.ST_SOLVED)[0]
    assert len(solved) >= 3
    horse = solver.model.model_type == 'animal_horse'
    col = dict(COL, poseB_jangles=COL['poseH']) if horse else COL
    dyn = solver.optimize_dynamics
    stats = {k: 0.0 for k in ('fullpose', 'markers', 'data/bound') + lib.ERR_NAMES[1:]}
    checked = {k: 0 for k in ('velo', 'extrap_dmpl')}
    for i, f in enumerate(solved):
        prev = solved[:i][solved[:i] >= seg[f]]             # solved frames in front of f on f's own (emitted) trajectory
        st = res.status[f]
        has_velo, has_extrap = bool(st & lib.ST_HAS_VELO), bool(st & lib.ST_HAS_EXTRAP)
        if seq:
            assert has_velo == (len(prev) >= 2) and has_extrap == (dyn and len(prev) >= 1), (f, st)
        else:
            assert has_velo or len(prev) < 2
            assert has_extrap or not dyn or len(prev) < 1
        skip = set()
        velo_target = dmpl_target = None
        if has_velo:
            if len(prev) >= 2:
                p1, p2 = res.pose[prev[-1]], res.pose[prev[-2]]
                velo_target = p1 + (p1 - p2)
                checked['velo'] += 1
            else:
                skip.add('velo')
        if has_extrap:
            if len(prev) >= 1:
                dmpl_target = res.dmpls[prev[-1], :solver.n_dm].copy()
                checked['extrap_dmpl'] += 1
            else:
                skip.add('extrap_dmpl')
        # the reported state
        solver.pose[:] = res.pose[f]
        solver.trans[:] = res.trans[f]
        if solver.nd:
            solver.betas[solver.lin_ids] = res.dmpls[f, :pk.n_dmpl]
        vidx = np.nonzero(vis[f])[0]
        terms, _ = solver.frame_terms(len(vidx), velo_target, dmpl_target)
        if 'velo' in skip:                                  # active in the kernel, target unknown here: any target will do
            terms.append(['velo', (solver.wts['stageii_wt_velo'], res.pose[f])])
        if 'extrap_dmpl' in skip:
            terms.append(['extrap_dmpl', (6.0, res.dmpls[f, :solver.n_dm])])
        obj = stageii._Objective(solver, obs[f, vidx], vidx, terms, solver.step2_ids, solver.nd > 0)

        fp = solver.model.fullpose(res.pose[f])
        e = np.abs(res.fullpose[f] - fp).max()
        assert e <= tol['fullpose'], (f, 'fullpose', e)
        stats['fullpose'] = max(stats['fullpose'], e)

        mk = solver.evaluate(False)['markers']             # all M markers
        assert res.markers_sim[f].shape == mk.shape
        e = np.abs(res.markers_sim[f] - mk).max()
        assert e <= tol['markers'], (f, 'markers', e)
        stats['markers'] = max(stats['markers'], e)

        sse = obj.term_sse()
        got = res.errs[f]
        for c, k in enumerate(lib.ERR_NAMES):              # columns of inactive terms stay zero
            if not any(col[name] == c for name in sse):
                assert got[c] == 0.0, (f, k, got[c])
        for name, ref in sse.items():
            if name in skip:
                continue
            c = col[name]
            k = got[c]
            key = lib.ERR_NAMES[c]
            if name == 'data':
                wt = dict(terms)['data']
                n3 = 3 * len(vidx)
                rn = np.linalg.norm(mk[vidx] - obs[f, vidx])
                eps = EPS32 if precision == 'f32' else 2.0 ** -53
                delta = tol['markers'] + eps * np.abs(obs[f, vidx]).max()
                bound = wt ** 2 * (2 * rn * np.sqrt(n3) * delta + n3 * delta ** 2) + (n3 + 8) * eps * ref
                assert abs(k - ref) <= bound, (f, name, k, ref, bound)
                stats['data/bound'] = max(stats['data/bound'], abs(k - ref) / bound)
                continue
            if name == 'poseB' and hasattr(solver.prior, 'weights'):
                # max-mixture: the SSE of any component within the margin of the float64 minimum
                xb = solver.pose[solver.body_ids]
                wt = dict(terms)['poseB']
                en = np.array([(l ** 2).sum() - np.log(w) for l, w in zip(solver.prior.loglikelihoods(xb), solver.prior.weights)])
                cand = wt ** 2 * en[en <= en.min() + tol['margin'] * max(1.0, abs(en.min()))]
                assert np.isclose(wt ** 2 * en.min(), ref, rtol=1e-12, atol=0)
                rel = np.abs(k - cand).min() / max(abs(ref), 1e-300)
            else:
                rel = abs(k - ref) / max(abs(ref), 1e-300)
            assert rel <= tol['rel'][key], (f, name, k, ref, rel)
            stats[key] = max(stats[key], rel)
    stats.update({'checked_' + k: v for k, v in checked.items()})
    return stats


# ---- CPU twin: the single-thread host build of the device source, both precisions, every family -----------------------

@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH'])
def test_device_source_output_state_equals_float64_evaluation(cases, emu, name, precision):
    case = cases(name)
    res = emu(case, precision={'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision])
    st = same_state_errors(case, res, precision)
    assert st['checked_velo'] > 0
    assert st['checked_extrap_dmpl'] > 0 or not case['cfg'].moshpp.optimize_dynamics


# ---- the CUDA kernels ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH'])
def test_kernel_output_state_equals_float64_evaluation(cases, name, precision):
    case = cases(name)
    st = same_state_errors(case, gpu_solve(case, precision=precision), precision)
    print(name, precision, {k: float('%.2g' % v) for k, v in st.items()})
    assert st['checked_velo'] > 0


@pytest.mark.gpu
@pytest.mark.parametrize('switch', [('MOSH2_DEV_BIG', '1'), ('MOSH2_DEV_THREADS', '256'), ('MOSH2_DEV_THREADS', '128')])
@pytest.mark.parametrize('name', ['C2', 'CF'])
def test_f32_kernel_output_state_under_other_launch_layouts(cases, name, switch, monkeypatch):
    """The float32 forward pass with A and the Jacobian tiles in a global workspace, and with 256 or 128 threads instead
    of 384: other CTA_FOR partitions, warp roles and reduction trees, the same bounds."""
    case = cases(name)
    monkeypatch.setenv(*switch)
    res = gpu_solve(case, precision='f32')
    monkeypatch.delenv(switch[0])
    st = same_state_errors(case, res, 'f32')
    print(name, switch, {k: float('%.2g' % v) for k, v in st.items()})


def _chunk_job(case, precision, chunk_len, warmup):
    from moshpp_b200 import chmosh
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    model = lib.Model(pk, device=0)
    job = model.job(dense_obs(case)[0].shape[0], opts, chunk_len=chunk_len, chunk_warmup=warmup,
                    precision={'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision])
    return model, job


def _segments(ranges, F, resumed=()):
    """seg_start per frame: a chunk with its own warm-up starts a trajectory; a resumed chunk continues its predecessor's."""
    seg = np.zeros(F, dtype=np.int64)
    for c, (a, b) in enumerate(ranges):
        seg[a:b] = seg[ranges[c - 1][0]] if (c in resumed and c > 0) else a
    return seg


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_chunked_kernel_output_state_equals_float64_evaluation(cases, precision):
    from moshpp_b200 import chmosh
    case = cases('C2')
    obs, vis = dense_obs(case)
    model, job = _chunk_job(case, precision, 5, 2)
    try:
        res, _ = chmosh.solve_verified(job, obs, vis, tol=None)
        ranges = job.chunk_ranges()
        assert len(ranges) == 4 and ranges[1, 0] == 5
        st = same_state_errors(case, res, precision, seg_start=_segments(ranges, obs.shape[0]))
        # every chunk's first two emitted frames have unemitted predecessors; the rest are checked
        assert st['checked_velo'] == sum(max(0, b - a - 2) for a, b in ranges)
    finally:
        job.close()
        model.close()


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_repaired_kernel_output_state_equals_float64_evaluation(cases, precision):
    """After one repair round (solve_verified, zero tolerance): the resumed chunks continue from the rows in front of them,
    so their first frames' velocity targets come from emitted rows and are checked."""
    from moshpp_b200 import chmosh
    case = cases('C2')
    obs, vis = dense_obs(case)
    model, job = _chunk_job(case, precision, 3, 1)
    try:
        job.upload(obs, vis)                 # the first launch alone: which chunks the repair round takes
        job.launch()
        bad = np.nonzero(job.boundary_deltas().max(1) > 0)[0]
        take, last = [], -2
        for c in bad:
            if c - 1 != last:
                take.append(int(c))
                last = int(c)
        assert len(take) >= 2
        res, rep = chmosh.solve_verified(job, obs, vis, tol=(0.0, 0.0, 0.0, 0.0), max_rounds=1)
        assert rep['repaired_chunks'] == [len(take)]
        ranges = job.chunk_ranges()
        st = same_state_errors(case, res, precision, seg_start=_segments(ranges, obs.shape[0], resumed=take))
        n = ranges[:, 1] - ranges[:, 0]
        assert st['checked_velo'] == sum(n[c] if c in take else max(0, n[c] - 2) for c in range(len(ranges)))
    finally:
        job.close()
        model.close()


# ---- boundary_delta_kernel, bit for bit ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('name,chunk_len,n_chunks', [
    ('C2', 3, 6),      # the "other" group holds the finger PCA coefficients; 6 = 2 mod 4 chunks
    ('C3', 2, 5),      # a DMPL group; 5 = 1 mod 4
    ('C4', 5, 3),      # MANO: the body group is the root alone; 3 = 3 mod 4
    ('C2', 1, 16),     # four full blocks of four warps
])
def test_boundary_deltas_equal_numpy_bit_for_bit(cases, name, chunk_len, n_chunks, precision):
    """mosh2_job_boundary_deltas after a launch with a one-frame cold warm-up: per chunk the maxima of |warm-up state -
    emitted row| on the chunk's last warm-up frame over (root + body pose, other pose coefficients, translation, linear
    coefficients), recomputed in the kernel's arithmetic (difference in the compute type, then float32(|.|)).  Chunks
    without a warm-up frame (warm_f = -1) report zeros."""
    case = cases(name)
    obs, vis = dense_obs(case)
    model, job = _chunk_job(case, precision, chunk_len, 1)
    try:
        assert job.num_chunks == n_chunks
        job.upload(obs, vis)
        job.launch()
        got = job.boundary_deltas()
        x, wf = job.warm_states()
        res = job.download()
        pk = model.pk
        PR, nd, body = pk.p_red, pk.n_dmpl, min(pk.body_dof, 66)
        ct = np.float64 if precision == 'f64' else np.float32
        want = np.zeros((n_chunks, 4), dtype=np.float32)
        for c in range(n_chunks):
            f = wf[c]
            if f < 0:
                continue
            d = lambda a, b: np.abs((a.astype(ct) - b.astype(ct)).astype(np.float32))
            dp = d(x[c, 3:3 + PR], res.pose[f])
            groups = (dp[:body], dp[body:], d(x[c, :3], res.trans[f]), d(x[c, 3 + PR:], res.dmpls[f, :nd]))
            want[c] = [g.max() if g.size else 0.0 for g in groups]
        assert wf[0] == -1 and (wf[1:] >= 0).all()
        assert np.array_equal(got.astype(np.float32), want), (got, want)
        # every group the model has is exercised with a nonzero delta somewhere
        assert (want[1:, 0] > 0).any() and (want[1:, 2] > 0).any()
        assert (want[1:, 1] > 0).any() == (PR > body) and (want[1:, 3] > 0).any() == (nd > 0)
    finally:
        job.close()
        model.close()
