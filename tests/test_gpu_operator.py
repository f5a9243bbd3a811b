"""The wide-state operator UDE (B200UDE_MODEL_OPERATOR) on the GPU against the fp64 reference (operator_ref.py): warp-per-
trajectory Tsit5 (fixed step and adaptive) and RKC2, forward and interpolating adjoint, fp32 and fp64."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

ACTN = {0: "identity", 1: "tanh", 2: "rbf"}

# name: (widths, acts, D1 kind, D2 given)
SHAPES = {
    "npde_30_8_30": ((30, 8, 30), (1, 1), "npde", True),
    "d1": ((1, 4, 1), (1, 0), "rand", True),
    "d32": ((32, 16, 32), (1, 0), "rand", True),
    "d33_m7": ((33, 24, 7), (2, 1), "rand", True),
    "d64": ((64, 64, 64), (1, 0), "rand", True),
    "d2_null": ((12, 40, 5), (1, 0), "rand", False),
    "climate_node": ((16, 32, 64, 64, 32, 16), (1, 1, 1, 1, 0), "eye", False),
}


def make(name, seed=0):
    widths, acts, kind, d2 = SHAPES[name]
    d, m = widths[0], widths[-1]
    rng = np.random.default_rng(seed)
    if kind == "npde":
        D1, D2 = R.npde_ops()
        D1, D2 = D1 * 0.02, D2 * 0.05
    elif kind == "eye":
        D1, D2 = np.eye(d), None
    else:
        D1 = rng.normal(scale=1.0 / np.sqrt(m), size=(d, m))
        D2 = -np.eye(d) + rng.normal(scale=0.3 / np.sqrt(d), size=(d, d)) if d2 else None
    model = R.Model(widths, acts, D1, D2 if d2 else None)
    theta = R.glorot(widths, rng) + 0.05 * rng.normal(size=model.P)
    return model, theta, rng


def solver_for(model, dtype, N, dt=0.05, n_steps=20, save_every=1, **kw):
    import universal_differential_equations_b200 as ude
    chain = ude.FastChain(*[ude.FastDense(a, b, getattr(ude, ACTN[k])) for a, b, k in zip(model.widths[:-1], model.widths[1:], model.acts)])
    f = ude.OperatorUDE(chain, model.D1, model.D2)
    return ude.UDESolver(f, 0.0, dt, n_steps, save_every, max_trajectories=N, device="cuda:0", dtype=dtype, **kw)


def run(s, theta, u0, cot=None, data=None):
    dt = s.dtype
    s.set_params(torch.tensor(theta, dtype=dt, device="cuda"))
    st = torch.empty(u0.shape[1], dtype=torch.int32, device="cuda")
    out = s.forward(torch.tensor(u0, dtype=dt, device="cuda"), status=st)
    if data is not None:
        loss, g, gu = s.adjoint_l2(torch.tensor(data, dtype=dt, device="cuda"), want_grad_u0=True)
        torch.cuda.synchronize()
        return out.cpu().numpy(), st.cpu().numpy(), float(loss), g.cpu().numpy(), gu.cpu().numpy()
    g, gu = s.adjoint(torch.tensor(cot, dtype=dt, device="cuda"))
    torch.cuda.synchronize()
    return out.cpu().numpy(), st.cpu().numpy(), None, g.cpu().numpy(), gu.cpu().numpy()


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("solver", ["tsit5", "rkc2"])
def test_fixed_step_fp64_matches_reference(name, solver):
    import universal_differential_equations_b200 as ude
    model, theta, rng = make(name)
    N, dt, n = 3, 0.05, 12
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    kw = dict(alg=ude.RKC2(stages=6)) if solver == "rkc2" else {}
    s = solver_for(model, torch.float64, N, dt, n, 2, **kw)
    cot = rng.normal(size=(n // 2 + 1, model.d, N))
    out, st, _, g, gu = run(s, theta, u0, cot=cot)
    assert (st == 0).all()
    gref = np.zeros(model.P)
    for j in range(N):
        if solver == "rkc2":
            o, rec = R.rkc2_fixed(model, theta, u0[:, j], dt, n, 6, 2)
            gt, lam, _ = R.rkc2_adjoint(model, theta, rec, dt, n, 6, 2, cot[:, :, j])
        else:
            o, rec = R.tsit5_fixed(model, theta, u0[:, j], 0.0, dt, n, 2)
            gt, lam, _ = R.tsit5_fixed_adjoint(model, theta, rec, dt, n, 2, cot[:, :, j])
        gref += gt
        assert rel(out[:, :, j], o) < 1e-10
        assert rel(gu[:, j], lam) < 1e-10
    assert rel(g, gref) < 1e-10


@pytest.mark.parametrize("name", ["npde_30_8_30", "d33_m7", "d2_null"])
def test_fixed_step_fp32_within_fp32_bounds(name):
    model, theta, rng = make(name)
    N, dt, n = 5, 0.05, 12
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    data = rng.normal(scale=0.5, size=(n + 1, model.d, N))
    out, st, loss, g, gu = run(solver_for(model, torch.float32, N, dt, n), theta, u0, data=data)
    gref, lref = np.zeros(model.P), 0.0
    for j in range(N):
        o, rec = R.tsit5_fixed(model, theta, u0[:, j], 0.0, dt, n)
        gt, lam, l = R.tsit5_fixed_adjoint(model, theta, rec, dt, n, 1, data[:, :, j], fused=True)
        gref += gt
        lref += l
        assert rel(out[:, :, j], o) < 2e-5
        assert rel(gu[:, j], lam) < 1e-3
    assert abs(loss - lref) / lref < 1e-4 and rel(g, gref) < 1e-3


@pytest.mark.parametrize("name", ["npde_30_8_30", "d33_m7", "d64"])
@pytest.mark.parametrize("tol", [(1e-6, 1e-3), (1e-8, 1e-8)])
def test_adaptive_fp64_matches_reference(name, tol):
    model, theta, rng = make(name)
    N, save_dt, n_save = 4, 0.1, 11
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    s = solver_for(model, torch.float64, N, save_dt, n_save - 1, 1, adaptive=True, abstol=tol[0], reltol=tol[1], max_steps=4000)
    cot = rng.normal(size=(n_save, model.d, N))
    out, st, _, g, gu = run(s, theta, u0, cot=cot)
    assert (st == 0).all()
    gref = np.zeros(model.P)
    for j in range(N):
        o, rec, stj = R.tsit5_adaptive(model, theta, u0[:, j], 0.0, save_dt, n_save, tol[0], tol[1])
        gt, lam, _ = R.tsit5_adaptive_adjoint(model, theta, rec, 0.0, save_dt, n_save, o, cot[:, :, j])
        gref += gt
        assert rel(out[:, :, j], o) < 1e-9, (j, len(rec[0]))
        assert rel(gu[:, j], lam) < 1e-9
        assert accepted_steps(model, theta, u0[:, j], save_dt, n_save, tol) == len(rec[0])
    assert rel(g, gref) < 1e-9


def accepted_steps(model, theta, u0, save_dt, n_save, tol):
    """the kernel's accepted-step count of one trajectory, read through max_steps: the largest max_steps that fails (status 2)
    plus one, found by bisection (a solve with max_steps = n succeeds exactly when it needs at most n accepted steps)."""
    lo, hi = 0, 4000   # fails at lo (nothing accepted yet), succeeds at hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        s = solver_for(model, torch.float64, 1, save_dt, n_save - 1, 1, adaptive=True, abstol=tol[0], reltol=tol[1], max_steps=mid)
        st = run(s, theta, u0[:, None], cot=np.zeros((n_save, model.d, 1)))[1]
        lo, hi = (lo, mid) if st[0] == 0 else (mid, hi)
    return hi


@pytest.mark.parametrize("mode", ["tsit5", "adaptive", "rkc2"])
def test_trajectories_are_independent_and_runs_deterministic(mode):
    import universal_differential_equations_b200 as ude
    model, theta, rng = make("npde_30_8_30")
    N = 9
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    u0[:, 3] *= 3.0   # a different step count in the adaptive solve
    kw = {"tsit5": {}, "adaptive": dict(adaptive=True, abstol=1e-6, reltol=1e-3, max_steps=2000), "rkc2": dict(alg=ude.RKC2(stages=5))}[mode]
    dt = torch.float64
    s = solver_for(model, dt, N, 0.1, 10, 1, **kw)
    data = rng.normal(size=(11, model.d, N))
    a = run(s, theta, u0, data=data)
    b = run(s, theta, u0, data=data)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))
    s1 = solver_for(model, dt, 1, 0.1, 10, 1, **kw)
    for j in (0, 3, 8):
        c = run(s1, theta, u0[:, j:j + 1], data=data[:, :, j:j + 1])
        assert np.array_equal(c[0][:, :, 0], a[0][:, :, j]) and np.array_equal(c[4][:, 0], a[4][:, j])


def test_status_words_non_finite_and_max_steps():
    model, theta, rng = make("d32")
    u0 = rng.normal(scale=0.5, size=(model.d, 2))
    u0[:, 1] = np.nan
    out, st, _, _, _ = run(solver_for(model, torch.float64, 2, 0.05, 10), theta, u0, cot=np.zeros((11, model.d, 2)))
    assert st[0] == 0 and st[1] == 1
    u0[:, 1] = 0.1
    s = solver_for(model, torch.float64, 2, 0.1, 10, 1, adaptive=True, abstol=1e-12, reltol=1e-12, max_steps=3)
    out, st, _, _, _ = run(s, theta, u0, cot=np.zeros((11, model.d, 2)))
    assert (st == 2).all() and np.isnan(out[-1]).all()


def test_explicit_cotangent_is_linear_and_fused_l2_equals_it():
    model, theta, rng = make("d33_m7")
    N = 4
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    s = solver_for(model, torch.float64, N, 0.05, 10)
    c1, c2 = rng.normal(size=(11, model.d, N)), rng.normal(size=(11, model.d, N))
    _, _, _, g1, u1 = run(s, theta, u0, cot=c1)
    _, _, _, g2, u2 = run(s, theta, u0, cot=c2)
    _, _, _, g3, u3 = run(s, theta, u0, cot=2 * c1 - c2)
    assert rel(g3, 2 * g1 - g2) < 1e-11 and rel(u3, 2 * u1 - u2) < 1e-11
    data = rng.normal(size=(11, model.d, N))
    out, _, loss, gl, ul = run(s, theta, u0, data=data)
    _, _, _, ge, ue = run(s, theta, u0, cot=2 * (out - data))
    assert rel(gl, ge) < 1e-12 and rel(ul, ue) < 1e-12 and abs(loss - np.sum((out - data) ** 2)) < 1e-9 * loss


def test_concurrent_handles_on_two_streams():
    model, theta, rng = make("npde_30_8_30")
    model2, theta2, _ = make("d33_m7", seed=1)
    N = 64
    ua, ub = rng.normal(scale=0.5, size=(30, N)), rng.normal(scale=0.5, size=(33, N))
    sa, sb = solver_for(model, torch.float64, N, 0.05, 20), solver_for(model2, torch.float64, N, 0.05, 20)
    ra, rb = run(sa, theta, ua, cot=np.ones((21, 30, N))), run(sb, theta2, ub, cot=np.ones((21, 33, N)))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            oa = sa.forward(torch.tensor(ua, dtype=torch.float64, device="cuda"))
            ga = sa.adjoint(torch.ones((21, 30, N), dtype=torch.float64, device="cuda"))
        with torch.cuda.stream(s2):
            ob = sb.forward(torch.tensor(ub, dtype=torch.float64, device="cuda"))
            gb = sb.adjoint(torch.ones((21, 33, N), dtype=torch.float64, device="cuda"))
        torch.cuda.synchronize()
        outs.append((oa.cpu().numpy(), ga[0].cpu().numpy(), ob.cpu().numpy(), gb[0].cpu().numpy()))
    for oa, ga, ob, gb in outs:
        assert np.array_equal(oa, ra[0]) and np.array_equal(ga, ra[3]) and np.array_equal(ob, rb[0]) and np.array_equal(gb, rb[3])


def test_usage_errors():
    import ctypes as C
    import universal_differential_equations_b200 as ude
    from universal_differential_equations_b200 import _lib
    model, theta, rng = make("d32")
    s = solver_for(model, torch.float32, 4)
    L = _lib.lib()
    a = np.asfortranarray(model.D1, dtype=np.float32)
    assert L.b200ude_set_operators(s._h, None, None, _lib.HOST, None) == _lib.EINVAL
    other = ude.UDESolver(ude.NeuralODE(ude.FastChain(ude.FastDense(2, 4, ude.tanh), ude.FastDense(4, 2))), 0.0, 0.1, 5, device="cuda:0")
    assert L.b200ude_set_operators(other._h, a.ctypes.data, None, _lib.HOST, None) == _lib.EUNSUPPORTED
    # a handle without operators: forward is ESTATE
    h = C.c_void_p()
    import test_operator_oracle as T
    rc = L.b200ude_create(C.byref(T._desc(widths=(32, 16, 32), acts=(1, 0))), C.byref(h))
    assert rc == 0
    th = np.zeros(model.P, np.float32)
    assert L.b200ude_set_params(h, th.ctypes.data, model.P, _lib.HOST, None) == 0
    u = torch.zeros((32, 4), device="cuda")
    o = torch.zeros((11, 32, 4), device="cuda")
    assert L.b200ude_forward(h, u.data_ptr(), 4, o.data_ptr(), None, None) == _lib.ESTATE
    assert b"set_operators" in L.b200ude_last_error(h)
    L.b200ude_destroy(h)


def _smem(widths, es, warps):
    """operator_layout / operator_smem of k_operator.cu: the dynamic shared memory of a CTA with `warps` gradient vectors."""
    d, m, q = widths[0], widths[-1], 16 // es
    ops = (64 + (d | 1) * m + (d | 1) * d + q - 1) // q * q
    th = sum(a * (b | 1) + b for a, b in zip(widths[:-1], widths[1:]))
    P = sum(a * b + b for a, b in zip(widths[:-1], widths[1:]))
    return es * (ops + th + warps * (P + 1))


def _static_smem():
    """the kernels' static shared memory as create reports it in its refusal of an fp64 shape that cannot fit one warp."""
    import re
    from universal_differential_equations_b200 import _lib
    with pytest.raises(_lib.B200UDEError) as e:
        solver_for(R.Model((64,) * 4, (1,) * 3, np.eye(64)), torch.float64, 2, 0.05, 4)
    assert e.value.code == _lib.EUNSUPPORTED and "shared memory" in str(e.value)
    return int(re.search(r"\+ (\d+) B static", str(e.value)).group(1))


def _closest(es, warps, cap, above):
    """(d, h1, h2, d) chain whose CTA with `warps` gradient vectors needs the least bytes above `cap` (above=True), or the
    most bytes not above it: (bytes - cap, widths)"""
    best = None
    for d in range(1, 65):
        for h1 in range(1, 65):
            for h2 in range(1, 65):
                x = _smem((d, h1, h2, d), es, warps) - cap
                if (x > 0) == above and (best is None or abs(x) < abs(best[0])):
                    best = (x, (d, h1, h2, d))
    return best


def _runs_at(widths, dt):
    model = R.Model(widths, (1, 1, 0), np.random.default_rng(2).normal(scale=0.2, size=(widths[0], widths[-1])))
    N = 5   # more trajectories than warps per CTA: two CTAs
    s = solver_for(model, dt, N, 0.05, 4)
    th = R.glorot(widths, np.random.default_rng(0))
    u0 = np.random.default_rng(1).normal(scale=0.3, size=(widths[0], N))
    cot = np.ones((5, widths[0], N))
    out, st, _, g, gu = run(s, th, u0, cot=cot)
    gref = np.zeros(model.P)
    tol = 2e-5 if dt == torch.float32 else 1e-10
    for j in range(N):
        o, rec = R.tsit5_fixed(model, th, u0[:, j], 0.0, 0.05, 4)
        gt, lam, _ = R.tsit5_fixed_adjoint(model, th, rec, 0.05, 4, 1, cot[:, :, j])
        gref += gt
        assert rel(out[:, :, j], o) < tol and rel(gu[:, j], lam) < 50 * tol
    assert rel(g, gref) < 50 * tol


@pytest.mark.parametrize("dtype,warps", [(torch.float32, 4), (torch.float64, 4), (torch.float64, 1)])
def test_shared_memory_edge(dtype, warps):
    """The warp count is the largest (<= 4) whose staged operators, padded theta and gradient vectors fit the opt-in shared
    memory next to the kernels' static shared memory.  At the boundary of `warps` on both sides: the chain closest to the limit
    from below runs with `warps`, the one closest from above runs with one warp fewer (or, at one warp, is refused)."""
    from universal_differential_equations_b200 import _lib
    es = 8 if dtype == torch.float64 else 4
    cap = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - _static_smem()
    below, above = _closest(es, warps, cap, False), _closest(es, warps, cap, True)
    assert -4 * es <= below[0] <= 0 and 0 < above[0] <= 8 * es, (below, above)   # within a few elements of the limit
    _runs_at(below[1], dtype)
    if warps > 1:
        assert _smem(above[1], es, warps - 1) <= cap
        _runs_at(above[1], dtype)
    else:
        with pytest.raises(_lib.B200UDEError) as e:
            solver_for(R.Model(above[1], (1, 1, 0), np.eye(above[1][0])), dtype, 2, 0.05, 4)
        assert e.value.code == _lib.EUNSUPPORTED and f"{_smem(above[1], es, 1)} B dynamic" in str(e.value)


def test_npde_script_transcribed():
    """Glorot init, adaptive Tsit5 at (1e-6, 1e-3) against the tight truth, BFGS; then ROCK2 in fp32 and the t = 10 RKC2 solve."""
    import universal_differential_equations_b200 as ude
    D1, D2 = R.npde_ops()
    saveat = np.linspace(0, 1.5, 30)
    truth = R.npde_truth(saveat)
    u0 = R.npde_u0()
    rng = np.random.default_rng(0)
    chain = ude.FastChain(ude.FastDense(30, 8, ude.tanh), ude.FastDense(8, 30, ude.tanh))
    f = ude.OperatorUDE(chain, D1, D2)
    th0 = R.glorot([30, 8, 30], rng)
    prob = ude.ODEProblem(f, u0, (0.0, 1.5))
    model = R.Model([30, 8, 30], [1, 1], D1, D2)

    def loss_of(dtype, alg, **kw):
        data = torch.tensor(truth.T, dtype=dtype, device="cuda")

        def loss(p):
            pred = ude.concrete_solve(prob, alg, torch.tensor(u0, dtype=dtype, device="cuda"), p, saveat=saveat, dtype=dtype, **kw)
            return ((data - pred) ** 2).sum()
        return loss

    # fp64: the gradient at theta0 against the CPU reference, then the first 5 BFGS iterations against a CPU replay of the same
    # sciml_train(BFGS) driven by the reference's loss and gradient
    loss64 = loss_of(torch.float64, ude.Tsit5(), abstol=1e-6, reltol=1e-3)
    p = torch.tensor(th0, dtype=torch.float64, device="cuda", requires_grad=True)
    L = loss64(p)
    L.backward()
    o, rec, st = R.tsit5_adaptive(model, th0, u0, 0.0, saveat[1], 30, 1e-6, 1e-3)
    gref, _, lref = R.tsit5_adaptive_adjoint(model, th0, rec, 0.0, saveat[1], 30, o, truth, fused=True)
    assert abs(float(L.detach()) - lref) < 1e-9 * lref and rel(p.grad.cpu().numpy(), gref) < 1e-8

    class RefLoss(torch.autograd.Function):
        @staticmethod
        def forward(ctx, th):
            t = th.detach().numpy()
            o, rec, _ = R.tsit5_adaptive(model, t, u0, 0.0, saveat[1], 30, 1e-6, 1e-3)
            g, _, l = R.tsit5_adaptive_adjoint(model, t, rec, 0.0, saveat[1], 30, o, truth, fused=True)
            ctx.g = torch.from_numpy(g)
            return torch.tensor(l, dtype=torch.float64)

        @staticmethod
        def backward(ctx, gl):
            return gl * ctx.g

    def trace():
        its = []
        return its, (lambda th, l: its.append((th.detach().cpu().numpy().copy(), l)) and False)

    gpu_its, cb_gpu = trace()
    cpu_its, cb_cpu = trace()
    res = ude.sciml_train(loss64, torch.tensor(th0, dtype=torch.float64, device="cuda"), ude.BFGS(), cb=cb_gpu, maxiters=5)
    ude.sciml_train(RefLoss.apply, torch.tensor(th0, dtype=torch.float64), ude.BFGS(), cb=cb_cpu, maxiters=5)
    assert len(gpu_its) == len(cpu_its) == 5
    e_th = max(rel(a[0], b[0]) for a, b in zip(gpu_its, cpu_its))
    e_l = max(abs(a[1] - b[1]) / b[1] for a, b in zip(gpu_its, cpu_its))
    print(f"MEASURED npde fp64 BFGS iterates 1-5 vs CPU replay: theta {e_th:.2e}, loss {e_l:.2e}; loss {gpu_its[0][1]:.4e} -> {res.minimum:.4e}")
    # measured on an H100: theta 1.2e-13, loss 6.5e-14 (the same accepted steps; round-off only)
    assert e_th < 1e-11 and e_l < 1e-11 and res.minimum < gpu_its[0][1]
    # fp32 with ROCK2(eigen_est = rho(D2)) at the save spacing: the loss decreases
    with pytest.warns(RuntimeWarning):
        alg = ude.ROCK2(eigen_est=191.7)
    loss32 = loss_of(torch.float32, alg, dt=saveat[1])
    l0 = float(loss32(torch.tensor(th0, dtype=torch.float32, device="cuda")))
    res32 = ude.sciml_train(loss32, torch.tensor(th0, dtype=torch.float32, device="cuda"), ude.BFGS(), maxiters=5)
    assert res32.minimum < l0
    # the solve of the trained model out to t = 10 (npde.jl:119-122) with RKC2: 194 steps of 10/194 (the save spacing rounded
    # down to divide 10), stage count from eigen_est; finite and on the reference
    th = res.minimizer.detach().cpu().numpy()
    n = int(np.ceil(10.0 / saveat[1]))
    dt10 = 10.0 / n
    S = alg.n_stages(dt10)
    s = ude.UDESolver(f, 0.0, dt10, n, 1, max_trajectories=1, device="cuda:0", alg=ude.RKC2(stages=S), dtype=torch.float64)
    s.set_params(torch.tensor(th, device="cuda"))
    out = s.forward(torch.tensor(u0[:, None], device="cuda")).cpu().numpy()[:, :, 0]
    ref, _ = R.rkc2_fixed(model, th, u0, dt10, n, S)
    assert n == 194 and abs(n * dt10 - 10.0) < 1e-12
    assert np.isfinite(out).all() and rel(out, ref) < 1e-10


@pytest.mark.parametrize("mode", ["tsit5", "adaptive"])
def test_fp32_host_entry_points_and_loss_weights(mode):
    """solve_host, loss_gradient_host, train_adam (its CUDA graph captures the new launches) and adjoint_l2_allreduce on one
    rank against the device-pointer calls; non-unit loss weights in the fused L2 against the reference."""
    import universal_differential_equations_b200 as ude
    model, theta, rng = make("d2_null")
    w = rng.uniform(0.2, 2.0, model.d)
    model.lossw = w
    N = 6
    u0 = rng.normal(scale=0.5, size=(model.d, N)).astype(np.float32)
    data = rng.normal(scale=0.5, size=(11, model.d, N)).astype(np.float32)
    kw = dict(adaptive=True, abstol=1e-6, reltol=1e-3, max_steps=500) if mode == "adaptive" else {}
    s = solver_for(model, torch.float32, N, 0.1, 10, 1, loss_weights=list(w), **kw)
    th32 = theta.astype(np.float32)
    out, st, loss, g, gu = run(s, th32.astype(np.float64), u0, data=data)
    # the fused L2 with weights against the fp64 reference
    lref, gref = 0.0, np.zeros(model.P)
    for j in range(N):
        if mode == "adaptive":
            o, rec, _ = R.tsit5_adaptive(model, th32.astype(np.float64), u0[:, j], 0.0, 0.1, 11, 1e-6, 1e-3)
            gt, _, l = R.tsit5_adaptive_adjoint(model, th32.astype(np.float64), rec, 0.0, 0.1, 11, o, data[:, :, j], fused=True)
        else:
            o, rec = R.tsit5_fixed(model, th32.astype(np.float64), u0[:, j], 0.0, 0.1, 10)
            gt, _, l = R.tsit5_fixed_adjoint(model, th32.astype(np.float64), rec, 0.1, 10, 1, data[:, :, j], fused=True)
        lref += l
        gref += gt
    assert abs(loss - lref) / lref < 1e-4 and rel(g, gref) < 1e-3
    # host-buffer entry points: the same numbers
    oh, sth = s.solve_host(th32, u0)
    assert np.array_equal(oh, out) and (sth == st).all()
    lh, gh, guh = s.loss_gradient_host(th32, u0, data, grad_u0=np.empty((model.d, N), np.float32))
    assert abs(lh - loss) <= 1e-6 * loss and rel(gh, g) < 1e-6 and rel(guh, gu) < 1e-6
    # adjoint_l2_allreduce on a one-rank group equals adjoint_l2 (fixed grid: the all-reduce path refuses adaptive handles)
    if mode == "tsit5":
        s.peer_attach(0, 1, s.peer_export())
        s.set_params(torch.tensor(th32, device="cuda"))
        s.forward(torch.tensor(u0, device="cuda"))
        la, ga, _ = s.adjoint_l2_allreduce(torch.tensor(data, device="cuda"))
        torch.cuda.synchronize()
        assert abs(float(la) - loss) <= 1e-6 * loss and rel(ga.cpu().numpy(), g) < 1e-6
        s.peer_detach()
    # train_adam (graph replay) against forward + adjoint_l2 + adam_step issued one by one
    opt = ude.ADAM(0.01)
    s.set_params(torch.tensor(th32, device="cuda"))
    s.adam_reset()
    ud, dd = torch.tensor(u0, device="cuda"), torch.tensor(data, device="cuda")
    hist = s.train_adam(opt, ud, dd, 4).cpu().numpy()
    th_graph = s.get_params().cpu().numpy()
    s.set_params(torch.tensor(th32, device="cuda"))
    s.adam_reset()
    steps = []
    for _ in range(4):
        s.forward(ud)
        l, gg, _ = s.adjoint_l2(dd)
        steps.append(float(l))
        s.adam_step(opt, gg)
    torch.cuda.synchronize()
    assert np.allclose(hist, steps, rtol=1e-6, atol=0) and hist[-1] < hist[0]
    assert rel(th_graph, s.get_params().cpu().numpy()) < 1e-6
