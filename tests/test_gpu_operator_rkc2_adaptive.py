"""Adaptive RKC2 on the operator UDE (operator.cuh, kernels 7 and 8) on the GPU against the fp64 reference
(operator_rkc2_adaptive_ref.py): forward, replay adjoint and accepted-step counts in fp64 and fp32, determinism, status words,
the loss paths, and Climate/NeuralPDE/npde.jl with ROCK2(eigen_est = 191.7) and no dt."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402
import operator_rkc2_adaptive_ref as A  # noqa: E402
from test_gpu_operator import make, rel, run, solver_for  # noqa: E402

pytestmark = pytest.mark.gpu

SAVE_DT, N_SAVE = 0.1, 11


def ark(model, dtype, N, tol, rho, max_steps=4000, stages=None, **kw):
    import universal_differential_equations_b200 as ude
    return solver_for(model, dtype, N, SAVE_DT, N_SAVE - 1, 1, alg=ude.RKC2(stages=stages, eigen_est=rho), adaptive=True,
                      abstol=tol[0], reltol=tol[1], max_steps=max_steps, **kw)


def accepted_steps(model, theta, u0, tol, rho):
    """the kernel's accepted-step count of one trajectory, read through max_steps as test_gpu_operator.accepted_steps does."""
    lo, hi = 0, 4000
    while hi - lo > 1:
        mid = (lo + hi) // 2
        st = run(ark(model, torch.float64, 1, tol, rho, max_steps=mid), theta, u0[:, None], cot=np.zeros((N_SAVE, model.d, 1)))[1]
        lo, hi = (lo, mid) if st[0] == 0 else (mid, hi)
    return hi


CASES = [("npde_30_8_30", 191.7), ("npde_30_8_30", 218.0), ("d1", 191.7), ("d33_m7", 191.7), ("d64", 218.0), ("d2_null", 191.7),
         ("climate_node", 191.7)]


@pytest.mark.parametrize("name,rho", CASES)
@pytest.mark.parametrize("tol", [(1e-6, 1e-3), (1e-4, 1e-2)])
def test_fp64_matches_reference(name, rho, tol):
    model, theta, rng = make(name)
    N = 3
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    cot = rng.normal(size=(N_SAVE, model.d, N))
    out, st, _, g, gu = run(ark(model, torch.float64, N, tol, rho), theta, u0, cot=cot)
    assert (st == 0).all()
    gref = np.zeros(model.P)
    for j in range(N):
        o, rec, stj = A.rkc2_adaptive(model, theta, u0[:, j], 0.0, SAVE_DT, N_SAVE, tol[0], tol[1], rho)
        gt, lam, _ = A.rkc2_adaptive_adjoint(model, theta, rec, 0.0, SAVE_DT, N_SAVE, o, cot[:, :, j])
        assert stj == 0
        gref += gt
        assert rel(out[:, :, j], o) < 1e-9, (j, len(rec[3]))
        assert rel(gu[:, j], lam) < 1e-9
        if j == 0:
            assert accepted_steps(model, theta, u0[:, j], tol, rho) == len(rec[3])
    assert rel(g, gref) < 1e-9


@pytest.mark.parametrize("name", ["npde_30_8_30", "d33_m7", "d2_null"])
def test_fp32_within_fp32_bounds(name):
    model, theta, rng = make(name)
    N = 4
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    data = rng.normal(scale=0.5, size=(N_SAVE, model.d, N))
    th32 = theta.astype(np.float32).astype(np.float64)
    out, st, loss, g, gu = run(ark(model, torch.float32, N, (1e-6, 1e-3), 191.7), th32, u0.astype(np.float32), data=data)
    assert (st == 0).all()
    gref, lref = np.zeros(model.P), 0.0
    for j in range(N):
        u0j = u0[:, j].astype(np.float32).astype(np.float64)
        o, rec, _ = A.rkc2_adaptive(model, th32, u0j, 0.0, SAVE_DT, N_SAVE, 1e-6, 1e-3, 191.7)
        gt, lam, l = A.rkc2_adaptive_adjoint(model, th32, rec, 0.0, SAVE_DT, N_SAVE, o, data[:, :, j].astype(np.float32), fused=True)
        gref += gt
        lref += l
        assert rel(out[:, :, j], o) < 2e-5
        assert rel(gu[:, j], lam) < 1e-3
    assert abs(loss - lref) / lref < 1e-4 and rel(g, gref) < 1e-3


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_trajectories_are_independent_and_runs_deterministic(dtype):
    model, theta, rng = make("npde_30_8_30")
    N = 9
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    u0[:, 3] *= 3.0   # a different step sequence
    s = ark(model, dtype, N, (1e-6, 1e-3), 191.7)
    data = rng.normal(size=(N_SAVE, model.d, N))
    a = run(s, theta, u0, data=data)
    b = run(s, theta, u0, data=data)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))
    s1 = ark(model, dtype, 1, (1e-6, 1e-3), 191.7)
    for j in (0, 3, 8):
        c = run(s1, theta, u0[:, j:j + 1], data=data[:, :, j:j + 1])
        assert np.array_equal(c[0][:, :, 0], a[0][:, :, j]) and np.array_equal(c[4][:, 0], a[4][:, j])


def test_max_steps_status_and_nan_saves_leave_other_trajectories_alone():
    model, theta, rng = make("npde_30_8_30")
    u0 = rng.normal(scale=0.5, size=(model.d, 3))
    tol = (1e-6, 1e-3)
    u0[:, 1] *= 4.0   # needs more steps than the others
    counts = [len(A.rkc2_adaptive(model, theta, u0[:, j], 0.0, SAVE_DT, N_SAVE, tol[0], tol[1], 191.7)[1][3]) for j in range(3)]
    cap = max(counts[0], counts[2])
    assert counts[1] > cap, counts
    cot = np.zeros((N_SAVE, model.d, 3))
    out, st, _, _, _ = run(ark(model, torch.float64, 3, tol, 191.7, max_steps=cap), theta, u0, cot=cot)
    assert st[0] == 0 and st[1] == 2 and st[2] == 0
    assert np.isnan(out[-1, :, 1]).all() and np.isfinite(out[:, :, [0, 2]]).all()
    ref, _, _, _, _ = run(ark(model, torch.float64, 3, tol, 191.7), theta, u0, cot=cot)
    assert np.array_equal(out[:, :, [0, 2]], ref[:, :, [0, 2]])
    o, _, stj = A.rkc2_adaptive(model, theta, u0[:, 1], 0.0, SAVE_DT, N_SAVE, tol[0], tol[1], 191.7, max_steps=cap)
    assert stj == 2 and np.array_equal(np.isnan(o), np.isnan(out[:, :, 1]))


def test_fused_l2_equals_the_explicit_cotangent():
    model, theta, rng = make("d33_m7")
    N = 4
    u0 = rng.normal(scale=0.5, size=(model.d, N))
    s = ark(model, torch.float64, N, (1e-6, 1e-3), 191.7)
    data = rng.normal(size=(N_SAVE, model.d, N))
    out, _, loss, gl, ul = run(s, theta, u0, data=data)
    _, _, _, ge, ue = run(s, theta, u0, cot=2 * (out - data))
    assert rel(gl, ge) < 1e-12 and rel(ul, ue) < 1e-12 and abs(loss - np.sum((out - data) ** 2)) < 1e-9 * loss


def test_fp32_host_entry_points_train_adam_and_allreduce_refusal():
    import universal_differential_equations_b200 as ude
    from universal_differential_equations_b200 import _lib
    model, theta, rng = make("d2_null")
    w = rng.uniform(0.2, 2.0, model.d)
    model.lossw = w
    N = 6
    u0 = rng.normal(scale=0.5, size=(model.d, N)).astype(np.float32)
    data = rng.normal(scale=0.5, size=(N_SAVE, model.d, N)).astype(np.float32)
    s = ark(model, torch.float32, N, (1e-6, 1e-3), 191.7, max_steps=500, loss_weights=list(w))
    th32 = theta.astype(np.float32)
    out, st, loss, g, gu = run(s, th32.astype(np.float64), u0, data=data)
    lref, gref = 0.0, np.zeros(model.P)
    for j in range(N):
        o, rec, _ = A.rkc2_adaptive(model, th32.astype(np.float64), u0[:, j], 0.0, SAVE_DT, N_SAVE, 1e-6, 1e-3, 191.7)
        gt, _, l = A.rkc2_adaptive_adjoint(model, th32.astype(np.float64), rec, 0.0, SAVE_DT, N_SAVE, o, data[:, :, j], fused=True)
        lref += l
        gref += gt
    assert abs(loss - lref) / lref < 1e-4 and rel(g, gref) < 1e-3
    oh, sth = s.solve_host(th32, u0)
    assert np.array_equal(oh, out) and (sth == st).all()
    lh, gh, guh = s.loss_gradient_host(th32, u0, data, grad_u0=np.empty((model.d, N), np.float32))
    assert abs(lh - loss) <= 1e-6 * loss and rel(gh, g) < 1e-6 and rel(guh, gu) < 1e-6
    s.peer_attach(0, 1, s.peer_export())
    with pytest.raises(_lib.B200UDEError) as e:
        s.adjoint_l2_allreduce(torch.tensor(data, device="cuda"))
    assert e.value.code == _lib.EUNSUPPORTED
    s.peer_detach()
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


def test_npde_script_with_rock2_and_no_dt():
    """npde.jl's training loss concrete_solve(prob, ROCK2(eigen_est = ...), u0, p; saveat) at the default tolerances: fp64 loss and
    gradient at theta0 and 5 BFGS iterates against a CPU replay driven by the reference; fp32 runs and descends; then the t = 10
    solve at (1e-4, 1e-2) on the save grid 10/194 against the reference."""
    import universal_differential_equations_b200 as ude
    D1, D2 = R.npde_ops()
    saveat = np.linspace(0, 1.5, 30)
    truth = R.npde_truth(saveat)
    u0 = R.npde_u0()
    chain = ude.FastChain(ude.FastDense(30, 8, ude.tanh), ude.FastDense(8, 30, ude.tanh))
    f = ude.OperatorUDE(chain, D1, D2)
    th0 = R.glorot([30, 8, 30], np.random.default_rng(0))
    prob = ude.ODEProblem(f, u0, (0.0, 1.5))
    model = R.Model([30, 8, 30], [1, 1], D1, D2)
    with pytest.warns(RuntimeWarning) if not ude.ROCK2._warned else _nullcontext():
        alg = ude.ROCK2(eigen_est=191.7)

    def loss_of(dtype):
        data = torch.tensor(truth.T, dtype=dtype, device="cuda")

        def loss(p):
            pred = ude.concrete_solve(prob, alg, torch.tensor(u0, dtype=dtype, device="cuda"), p, saveat=saveat, dtype=dtype)
            return ((data - pred) ** 2).sum()
        return loss

    loss64 = loss_of(torch.float64)
    p = torch.tensor(th0, dtype=torch.float64, device="cuda", requires_grad=True)
    L = loss64(p)
    L.backward()

    def ref(t):
        o, rec, st = A.rkc2_adaptive(model, t, u0, 0.0, saveat[1], 30, 1e-6, 1e-3, 191.7)
        assert st == 0
        return A.rkc2_adaptive_adjoint(model, t, rec, 0.0, saveat[1], 30, o, truth, fused=True)

    gref, _, lref = ref(th0)
    assert abs(float(L.detach()) - lref) < 1e-9 * lref and rel(p.grad.cpu().numpy(), gref) < 1e-9

    class RefLoss(torch.autograd.Function):
        @staticmethod
        def forward(ctx, th):
            g, _, l = ref(th.detach().numpy())
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
    print(f"MEASURED npde adaptive RKC2 fp64 BFGS iterates 1-5 vs CPU replay: theta {e_th:.2e}, loss {e_l:.2e}; "
          f"loss {gpu_its[0][1]:.4e} -> {res.minimum:.4e}")
    assert e_th < 1e-9 and e_l < 1e-9 and res.minimum < gpu_its[0][1]
    # fp32: the same call runs adaptively and the loss decreases
    loss32 = loss_of(torch.float32)
    l0 = float(loss32(torch.tensor(th0, dtype=torch.float32, device="cuda")))
    assert abs(l0 - lref) < 1e-3 * lref
    res32 = ude.sciml_train(loss32, torch.tensor(th0, dtype=torch.float32, device="cuda"), ude.BFGS(), maxiters=5)
    assert res32.minimum < l0
    # the solve out to t = 10 (npde.jl:119-123): solve(prob2, ROCK2(eigen_est = ...), saveat, abstol = 1e-4, reltol = 1e-2)
    th = res.minimizer.detach().cpu().numpy()
    n = int(np.ceil(10.0 / saveat[1]))
    sv = np.linspace(0.0, 10.0, n + 1)
    out = ude.concrete_solve(ude.ODEProblem(f, u0, (0.0, 10.0)), alg, u0, torch.tensor(th, device="cuda"), saveat=sv,
                             abstol=1e-4, reltol=1e-2, dtype=torch.float64).cpu().numpy()
    o, rec, st = A.rkc2_adaptive(model, th, u0, 0.0, sv[1], n + 1, 1e-4, 1e-2, 191.7)
    assert n == 194 and st == 0 and np.isfinite(out).all()
    # The trained closure amplifies perturbations from t ~ 4 on: the reference itself moves by up to ~1e-4 when theta moves by
    # 1e-14 (relative), with the same accepted steps.  So the bound per save is 1e-9 plus ten times that envelope (running max
    # over theta (1 +- 1e-14)); before t ~ 4 it is 1e-9.  Measured on an H100: at most 2.4 x the envelope.
    env = np.zeros(n + 1)
    for e in (1e-14, -1e-14):
        o2, rec2, _ = A.rkc2_adaptive(model, th * (1 + e), u0, 0.0, sv[1], n + 1, 1e-4, 1e-2, 191.7)
        assert len(rec2[3]) == len(rec[3])
        env = np.maximum(env, np.abs(o2 - o).max(1))
    env = np.maximum.accumulate(env)
    dev = np.abs(out.T - o).max(1)
    print(f"MEASURED npde t = 10: max deviation / (1e-9 + envelope) = {(dev / (1e-9 + env)).max():.2f}; {len(rec[3])} accepted steps")
    assert (dev <= 1e-9 + 10 * env).all() and (dev[sv < 4.0] < 1e-9).all()
    for ms in (len(rec[3]) - 1, len(rec[3])):   # the kernel's accepted-step count is the reference's
        s = ude.UDESolver(f, 0.0, sv[1], n, 1, max_trajectories=1, device="cuda:0", alg=alg, adaptive=True, abstol=1e-4, reltol=1e-2,
                          max_steps=ms, dtype=torch.float64)
        s.set_params(torch.tensor(th, device="cuda"))
        st = torch.empty(1, dtype=torch.int32, device="cuda")
        s.forward(torch.tensor(u0[:, None], device="cuda"), status=st)
        assert int(st.cpu()[0]) == (2 if ms < len(rec[3]) else 0)


class _nullcontext:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
