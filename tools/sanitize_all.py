"""Small invocations of every kernel family (for compute-sanitizer memcheck)."""
import sys, numpy as np, torch
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import universal_differential_equations_b200 as ude
from helpers import glorot_theta, synthetic_ensemble

def run(name, f, theta, u0, y, dt, n_steps, every, **kw):
    s = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=u0.shape[1], **kw)
    s.set_params(torch.from_numpy(theta.astype(np.float32)).cuda())
    out = s.forward(torch.from_numpy(u0).cuda())
    L, g, gu = s.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
    l2 = s.train_adam(ude.ADAM(0.01), torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda(), 3)
    torch.cuda.synchronize()
    print(name, float(L), float(g.abs().sum()), l2.cpu().numpy())
    s.close()

rng = np.random.default_rng(0)
N = 300
u0, y = synthetic_ensemble(N)
lv32 = ude.LotkaVolterraUDE(ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2)))
run("lv32", lv32, glorot_theta((2, 32, 32, 2), seed=1), u0, y, 0.1, 30, 1)
run("lv32-adaptive-tc", lv32, glorot_theta((2, 32, 32, 2), seed=1), u0, y, 0.1, 30, 1, adaptive=True, abstol=1e-5, reltol=1e-5, max_steps=200)
run("lv32-discrete", lv32, glorot_theta((2, 32, 32, 2), seed=1), u0, y, 0.1, 30, 1, sensealg=ude.ForwardDiffSensitivity())
lv5 = ude.LotkaVolterraUDE(ude.FastChain(ude.FastDense(2, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 5, ude.tanh), ude.FastDense(5, 2)), trainable_rates=2)
run("lv5p2", lv5, np.concatenate([[1.3, 1.8], glorot_theta((2, 5, 5, 5, 2), seed=2)]), u0, y, 0.1, 30, 1)
run("lv5p2-discrete", lv5, np.concatenate([[1.3, 1.8], glorot_theta((2, 5, 5, 5, 2), seed=2)]), u0, y, 0.1, 30, 1, sensealg=ude.ForwardDiffSensitivity())
gen = ude.LotkaVolterraUDE(ude.FastChain(ude.FastDense(2, 7, ude.tanh), ude.FastDense(7, 2)))
run("generic", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1)
run("adaptive", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, adaptive=True, abstol=1e-5, reltol=1e-5, max_steps=200)
run("vern7", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7())
run("vern7-adaptive", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7(), adaptive=True, abstol=1e-5, reltol=1e-5, max_steps=200)
# Vern7 dense output (vern7_dense.cuh): fixed-step adjoint, adaptive forward and replay adjoint
run("vern7-dense", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7(dense=True))
run("vern7-dense-adaptive", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7(dense=True), adaptive=True, abstol=1e-5,
    reltol=1e-5, max_steps=200)
# discrete adjoint (discrete_adjoint.cuh): fp32 through every entry point, fp64 through forward / adjoint_l2
fd = ude.ForwardDiffSensitivity()
run("generic-discrete", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, sensealg=fd)
run("vern7-discrete", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7(), sensealg=fd)
run("vern7-adaptive-discrete", gen, glorot_theta((2, 7, 2), seed=3), u0, y, 0.1, 30, 1, alg=ude.Vern7(), adaptive=True, abstol=1e-5, reltol=1e-5,
    max_steps=200, sensealg=fd)
for alg, adaptive in ((ude.Tsit5(), False), (ude.Vern7(), False), (ude.Vern7(), True)):
    s = ude.UDESolver(gen, 0.0, 0.1, 30, 1, max_trajectories=N, alg=alg, adaptive=adaptive, abstol=1e-6, reltol=1e-6, sensealg=fd, dtype=torch.float64)
    s.set_params(torch.from_numpy(glorot_theta((2, 7, 2), seed=3).astype(np.float64)).cuda())
    s.forward(torch.from_numpy(u0.astype(np.float64)).cuda())
    L, g, gu = s.adjoint_l2(torch.from_numpy(y.astype(np.float64)).cuda(), want_grad_u0=True)
    torch.cuda.synchronize()
    print("f64-discrete", type(alg).__name__, adaptive, float(L), float(g.abs().sum()))
    s.close()
Ns = 300
S0 = 14e6
us = np.zeros((7, Ns), np.float32); us[0] = 0.9 * S0; us[1:4] = rng.uniform(0, 50, (3, Ns)); us[4] = S0
ys = rng.uniform(0, 100, (8, 7, Ns)).astype(np.float32)
seir = ude.SEIRExposureUDE(ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1)))
run("seir64", seir, glorot_theta((3, 64, 64, 1), seed=2), us, ys, 0.25, 28, 4, loss_weights=[0, 1, 1, 1, 0, 0, 0])
run("seir64-vern7-adaptive-discrete", seir, glorot_theta((3, 64, 64, 1), seed=2), us, ys, 1.0, 7, 1, loss_weights=[0, 1, 1, 1, 0, 0, 0], alg=ude.Vern7(),
    adaptive=True, abstol=1e-4, reltol=1e-4, max_steps=128, sensealg=ude.ForwardDiffSensitivity())
run("seir64-adaptive-tc", seir, glorot_theta((3, 64, 64, 1), seed=2), us, ys, 1.0, 7, 1, loss_weights=[0, 1, 1, 1, 0, 0, 0], adaptive=True, abstol=1e-4, reltol=1e-4, max_steps=128)
node = ude.SEIRNeuralODE(ude.FastChain(ude.FastDense(7, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 7)))
run("seir-node", node, 0.3 * glorot_theta((7, 64, 64, 64, 7), seed=6), us[:, :40].copy(), ys[:, :, :40].copy(), 0.25, 28, 4, loss_weights=[0, 1, 1, 1, 0, 0, 0])
for nx, n in ((26, 7), (27, 5), (256, 3)):
    fk = ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)), nx)
    th = np.concatenate([glorot_theta((1, 16, 16, 1), seed=4), [1.1, -2.3, 0.9, 0.0, 0.01 * (nx - 1) ** 2]])
    x = np.linspace(0, 1, nx)
    uf = np.stack([np.exp(-((x - 0.5) / d) ** 2) for d in rng.uniform(0.05, 0.3, n)], axis=1).astype(np.float32)
    yf = np.repeat(uf[None], 6, axis=0)
    run(f"fkpp16 nx={nx}", fk, th, uf, yf, 2.5 / (16 * 0.01 * (nx - 1) ** 2), 40, 8)
    fk2 = ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 10, ude.tanh), ude.FastDense(10, 1)), nx)
    th2 = np.concatenate([glorot_theta((1, 10, 1), seed=4), [1.1, -2.3, 0.9, 0.0, 0.01 * (nx - 1) ** 2]])
    run(f"fkpp-generic nx={nx}", fk2, th2, uf, yf, 2.5 / (16 * 0.01 * (nx - 1) ** 2), 40, 8)
# the largest adjoint footprints of the runtime-shape kernels: fp32 at the 12 288-float constant bank (4 x 12 289 floats of shared
# memory per CTA), fp64 at 8-64-64-64-64-8 (2 x 13 577 doubles)
sys.path.insert(0, 'tests')
import envelope_cases as E
run("lv_bank", E.ude_form("lv_bank"), E.theta("lv_bank"), u0[:, :130].copy(), y[:, :, :130].copy(), 0.1, 30, 1)
s = ude.UDESolver(E.ude_form("node8_max"), 0.0, 0.05, 20, 2, max_trajectories=130, dtype=torch.float64)
s.set_params(torch.from_numpy(E.theta("node8_max")).cuda())
u8 = torch.from_numpy(E.u0("node8_max", 130)).cuda()
out8 = s.forward(u8)
L, g, gu = s.adjoint_l2(out8 + 0.1, want_grad_u0=True)
torch.cuda.synchronize()
print("node8_max f64", float(L), float(g.abs().sum()))
s.close()
# adaptive RKC2 on the operator UDE (operator.cuh kernels 7 and 8): npde.jl's 30-8-30 closure, stage count per step from eigen_est
import operator_ref as OR
D1, D2 = OR.npde_ops()
opf = ude.OperatorUDE(ude.FastChain(ude.FastDense(30, 8, ude.tanh), ude.FastDense(8, 30, ude.tanh)), D1, D2)
zo = OR.npde_grid()[1:31]
uo = np.exp(-200.0 * (zo[:, None] - rng.uniform(0.2, 0.8, 70)[None, :]) ** 2).astype(np.float32)
yo = np.repeat(uo[None], 11, axis=0)
tho = OR.glorot([30, 8, 30], np.random.default_rng(0))
run("operator-rkc2-adaptive f32", opf, tho, uo, yo, 0.15, 10, 1, alg=ude.RKC2(eigen_est=191.7), adaptive=True, max_steps=400)
s = ude.UDESolver(opf, 0.0, 0.15, 10, 1, max_trajectories=70, alg=ude.RKC2(eigen_est=191.7), adaptive=True, max_steps=400, dtype=torch.float64)
s.set_params(torch.from_numpy(tho).cuda())
s.forward(torch.from_numpy(uo.astype(np.float64)).cuda())
L, g, gu = s.adjoint_l2(torch.from_numpy(yo.astype(np.float64)).cuda(), want_grad_u0=True)
torch.cuda.synchronize()
print("operator-rkc2-adaptive f64", float(L), float(g.abs().sum()))
s.close()
print("ALL DONE")
