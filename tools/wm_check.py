"""Dev check of the warp-collective LV kernels (lv32_wm.cuh): parity vs the fp64 oracle and timings per family.
Run on an H100:  python tools/wm_check.py"""
import os, sys, json
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import universal_differential_equations_b200 as ude
from helpers import glorot_theta, synthetic_ensemble
from oracle import oracle as O

chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
f = ude.LotkaVolterraUDE(chain)
theta = glorot_theta((2, 32, 32, 2), seed=1)
m = O.lv_model()


def make(N, fwd, adj, G=1, R=0, **kw):
    os.environ["B200UDE_FWD_WM"] = str(fwd); os.environ["B200UDE_ADJ_WM"] = str(adj); os.environ["B200UDE_WM_G"] = str(G); os.environ["B200UDE_WM_R"] = str(R)
    return ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, **kw)


def parity(N, fwd, adj, G=1, R=0):
    u0, y = synthetic_ensemble(N)
    s = make(N, fwd, adj, G, R)
    s.set_params(torch.from_numpy(theta).cuda())
    st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = s.forward(torch.from_numpy(u0).cuda(), status=st)
    loss, g, gu = s.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
    torch.cuda.synchronize()
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
    o = out.cpu().numpy()
    r = dict(N=N, fwd=fwd, adj=adj, G=G, R=R, out=float((np.abs(o - out64) / (1 + np.abs(out64))).max()), loss=abs(float(loss) - l64) / l64,
             g=float(np.linalg.norm(g.cpu().numpy() - g64) / np.linalg.norm(g64)), gu=float(np.abs(gu.cpu().numpy() - gu64).max() / np.abs(gu64).max()),
             status=int((st != 0).sum()))
    # per-block relative errors of the gradient
    gg = g.cpu().numpy()
    for name, lo, hi in (("W1", 0, 64), ("b1", 64, 96), ("W2", 96, 1120), ("b2", 1120, 1152), ("W3", 1152, 1216), ("b3", 1216, 1218)):
        r["g_" + name] = float(np.linalg.norm(gg[lo:hi] - g64[lo:hi]) / np.linalg.norm(g64[lo:hi]))
    print(json.dumps(r)); sys.stdout.flush()
    s.close()


def timing(N, fwd, adj, G=1, R=0, reps=20):
    u0, y = synthetic_ensemble(N)
    s = make(N, fwd, adj, G, R)
    s.set_params(torch.from_numpy(theta).cuda())
    u0d, yd = torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda()
    out = torch.empty((31, 2, N), device="cuda")
    for _ in range(5):
        s.forward(u0d, out=out); s.adjoint_l2(yd)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tf = ta = 0.0
    for _ in range(reps):
        ev[0].record(); s.forward(u0d, out=out); ev[1].record(); s.adjoint_l2(yd); ev[2].record(); torch.cuda.synchronize()
        tf += ev[0].elapsed_time(ev[1]); ta += ev[1].elapsed_time(ev[2])
    print(json.dumps(dict(N=N, fwd=fwd, adj=adj, G=G, R=R, fwd_ms=round(tf / reps, 4), adj_ms=round(ta / reps, 4), Mtraj_s=round(N / ((tf + ta) / reps * 1e-3) / 1e6, 2))))
    sys.stdout.flush()
    s.close()


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("all", "parity"):
        for N in (1, 9, 257, 4097):
            parity(N, 1, 1, R=1)
        for N in (1, 17, 1000, 4097):
            parity(N, 1, 1, R=2)
        parity(1000, 1, 1, G=2, R=2)
    if what in ("all", "timing"):
        for N in (1024, 4096, 8192, 16384, 32768, 65536):
            for R in (1, 2):
                if (R == 1 and N > 8192) or (R == 2 and N < 4096):
                    continue
                timing(N, 1, 1, 1, R)
