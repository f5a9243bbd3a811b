"""Time one training iteration (forward + fused-L2 replay adjoint + reduce) of adaptive Tsit5 on the Fisher-KPP UPDE with the
checkpointed record (B200UDE_FLAG_CHECKPOINT) and with the full record, and report each handle's b200ude_device_bytes.

    python tools/fkpp_checkpoint_speed.py [--rounds 5] [--reps 10] [--warmup 3] [--big-reps 1] [--json out.json]

Cases, each in fp32 and fp64, max_steps = 2048 (K = 17): 26 points with the 1-5-5-5-1 rbf chain at N = 4096 on (0, 5), and 256
points with the 1-16-16-1 tanh chain at N = 1024 on (0, 0.2), D0 = 0.01 / dx^2, abstol 1e-6 / reltol 1e-3.  The two handles of
a case are timed in alternation over `rounds` rounds (CUDA events around `reps` back-to-back iterations after `warmup` untimed
ones); the median round is reported.  Then the checkpointed handle alone at 256 points, N = 65 536, fp32 (its full record would
not fit on an 80 GB card).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import universal_differential_equations_b200 as ude  # noqa: E402

MAX_STEPS = 2048


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _problem(Nx, widths, acts, N, seed=0):
    rng = np.random.default_rng(seed)
    chain = ude.FastChain(*[ude.FastDense(a, b, act) for a, b, act in zip(widths[:-1], widths[1:], acts)])
    theta = np.concatenate([ude.initial_params(chain, rng), [1.0, -2.0, 1.0, 0.0, 0.01 * (Nx - 1) ** 2]])
    x = np.linspace(0.0, 1.0, Nx)[:, None]
    d = rng.uniform(0.2, 0.6, N)[None, :]
    u0 = (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) / 2
    return ude.FisherKPPUDE(chain, Nx), theta, u0


class Iteration:
    def __init__(self, f, theta, u0, T, dtype, ckpt):
        N = u0.shape[1]
        self.solver = ude.UDESolver(f, 0.0, T / 10, 10, 1, max_trajectories=N, adaptive=True, abstol=1e-6, reltol=1e-3, max_steps=MAX_STEPS,
                                    dtype=dtype, sensealg=ude.InterpolatingAdjoint(checkpointing=ckpt))
        self.bytes = int(self.solver._L.b200ude_device_bytes(self.solver._h))
        self.solver.set_params(torch.as_tensor(theta, dtype=dtype, device="cuda"))
        self.u = torch.as_tensor(u0, dtype=dtype, device="cuda")
        self.st = torch.zeros(N, dtype=torch.int32, device="cuda")
        self.out = self.solver.forward(self.u, status=self.st)
        self.data = (0.9 * self.out).contiguous()
        self.gth = torch.empty(self.solver.P, dtype=dtype, device="cuda")
        self.loss = torch.empty(1, dtype=dtype, device="cuda")

    def __call__(self):
        self.solver.forward(self.u, out=self.out, status=self.st)
        self.solver.adjoint_l2(self.data, grad_theta=self.gth, loss=self.loss)

    def time(self, reps, warmup):
        for _ in range(warmup):
            self()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            self()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps

    def result(self):
        return self.out.cpu().numpy(), self.st.cpu().numpy(), self.loss.cpu().numpy(), self.gth.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--big-reps", type=int, default=1)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fkpp_checkpoint_speed: needs a CUDA device")
    name, power = _card()
    print(f"card: {name}, power limit {power}")
    rows = []
    cases = [(26, (1, 5, 5, 5, 1), ("rbf", "rbf", "rbf", "identity"), 4096, 5.0), (256, (1, 16, 16, 1), ("tanh", "tanh", "identity"), 1024, 0.2)]
    for Nx, widths, acts, N, T in cases:
        f, theta, u0 = _problem(Nx, widths, acts, N)
        for dtype in (torch.float32, torch.float64):
            its = {ck: Iteration(f, theta, u0, T, dtype, ck) for ck in (False, True)}
            ms = {False: [], True: []}
            for _ in range(a.rounds):
                for ck in (False, True):
                    ms[ck].append(its[ck].time(a.reps, a.warmup))
            r0, r1 = its[False].result(), its[True].result()
            same = all(np.array_equal(x, y, equal_nan=True) for x, y in zip(r0, r1))
            row = {"Nx": Nx, "N": N, "dtype": str(dtype).split(".")[-1], "ms_full": float(np.median(ms[False])),
                   "ms_ckpt": float(np.median(ms[True])), "ms_full_rounds": ms[False], "ms_ckpt_rounds": ms[True],
                   "bytes_full": its[False].bytes, "bytes_ckpt": its[True].bytes, "bitwise_equal": same, "status_ok": bool((r1[1] == 0).all())}
            row["overhead"] = row["ms_ckpt"] / row["ms_full"] - 1
            print(json.dumps(row), flush=True)
            rows.append(row)
            for it in its.values():
                it.solver.close()
            del its
            torch.cuda.empty_cache()
    f, theta, u0 = _problem(256, (1, 16, 16, 1), ("tanh", "tanh", "identity"), 65536)
    it = Iteration(f, theta, u0, 0.2, torch.float32, True)
    ms = it.time(a.big_reps, 1)
    row = {"Nx": 256, "N": 65536, "dtype": "float32", "ms_ckpt": ms, "bytes_ckpt": it.bytes, "status_ok": bool((it.st == 0).all())}
    print(json.dumps(row), flush=True)
    rows.append(row)
    it.solver.close()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": name, "power_limit": power, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
