"""GPU tests of the fused fp64 terminal-PDE kernels (csrc/bsde.cu) at the benchmarked size and in every variant b200ude_bsde_create
can select, against oracle/bsde_oracle.py.

The lock-free parts of the fused path -- the k_wgrad chunk ring refilled by its last reader, the persistent k_fused_backward CTAs
walking task group after task group, partial tiles, groups and CTAs -- only run at sizes well above those of tests/test_gpu_bsde.py.
Each size test below first asserts, from the launch shape mirrored in `geometry`, that the code path it exists for really runs.

Tolerances are those of tests/test_gpu_bsde.py: fp64 loss and u0(x0) relative 1e-10, gradient ||g - g_o|| / ||g_o|| 1e-9, the
whole vector and each parameter block on its own (the u0 net, then [W | b] of each z-net layer, so that one wrong layer of k_wgrad
cannot hide in the norm of the rest); fp32 loss 2e-4, gradient 2e-3.  Largest values measured on an H100 80GB HBM3 (700 W power
limit) over this file: fp64 loss 7.7e-16, u0 2.4e-16, gradient 4.7e-16, a parameter block 6.1e-16; fp32 library path loss 1.8e-8,
gradient 1.7e-7.  The numpy oracle took 3.0-3.3 s per iteration at 10 000 paths on that machine's CPU.
"""
import math
import time
from types import SimpleNamespace

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import bsde_oracle as bo  # noqa: E402

# Launch constants of csrc/bsde.cu.
WGR = 16      # WGR: tape rows per k_wgrad chunk
WGD = 4       # WGD: stages of the k_wgrad chunk ring; grid.x of k_wgrad = wg_splits = sm_count / 4
FWPC = 4      # FWPC: warps of a k_fused_backward CTA, one (step, 8-path tile) task each; grid = min(groups, 3 * sm_count)
FWF = 4       # FWF: warps of a k_fused_forward CTA (B200UDE_BSDE_PAIRS=0), one 8-path tile each
FP_TILES = 5  # FPW / 2: warp pairs of a k_fused_forward2 CTA (the default forward), one 8-path tile each

F64_TOL = dict(loss=1e-10, u0=1e-10, grad=1e-9)
F32_TOL = dict(loss=2e-4, grad=2e-3)

VARIANTS = {
    "default": {},
    "pairs0": {"BSDE_PAIRS": "0"},
    "wgrad0": {"BSDE_WGRAD": "0"},
    "pairs0_wgrad0": {"BSDE_PAIRS": "0", "BSDE_WGRAD": "0"},
    "fused0": {"BSDE_FUSED": "0"},
}


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def geometry(M, N, sm_count):
    """Launch shape of the fused sweeps for M paths and N steps, as fused_sweeps() and loss_gradient() in csrc/bsde.cu compute it."""
    tiles = -(-M // 8)
    splits = max(sm_count // 4, 1)
    chunks = -(-N * M // WGR)
    tasks = tiles * N
    groups = -(-tasks // FWPC)
    bwd_ctas = min(groups, 3 * sm_count)
    fwd_ctas, fwd2_ctas = -(-tiles // FWF), -(-tiles // FP_TILES)
    return SimpleNamespace(
        tiles=tiles, last_tile_paths=M - 8 * (tiles - 1),
        wg_splits=splits, wg_chunks=[chunks * (b + 1) // splits - chunks * b // splits for b in range(splits)],
        bwd_tasks=tasks, bwd_groups=groups, bwd_ctas=bwd_ctas, bwd_rounds=-(-groups // bwd_ctas), bwd_last_group_tasks=tasks - FWPC * (groups - 1),
        fwd_last_cta_tiles=tiles - FWF * (fwd_ctas - 1), fwd2_last_cta_tiles=tiles - FP_TILES * (fwd2_ctas - 1))


def _show(tag, g):
    print(f"[{tag}] {g.tiles} tiles (last {g.last_tile_paths} paths); k_wgrad {g.wg_splits} CTAs x {min(g.wg_chunks)}..{max(g.wg_chunks)} chunks; "
          f"k_fused_backward {g.bwd_tasks} tasks in {g.bwd_groups} groups on {g.bwd_ctas} CTAs ({g.bwd_rounds} rounds, last group "
          f"{g.bwd_last_group_tasks} tasks); last forward CTA {g.fwd_last_cta_tiles}/{FWF} tiles, last forward2 CTA "
          f"{g.fwd2_last_cta_tiles}/{FP_TILES} tiles")


def _problem(ude, d, hls, x0):
    prob = ude.TerminalPDEProblem(ude.HJBTerminal(0.5, 0.5), ude.HJBNonlinearity(1.0), ude.ZeroDrift(), ude.ConstantDiffusion(math.sqrt(2.0)), x0, (0.0, 1.0))
    u0 = ude.Chain(ude.Dense(d, hls, ude.relu), ude.Dense(hls, hls, ude.relu), ude.Dense(hls, 1))
    sg = ude.Chain(ude.Dense(d + 1, hls, ude.relu), ude.Dense(hls, hls, ude.relu), ude.Dense(hls, hls, ude.relu), ude.Dense(hls, d))
    return prob, ude.NNPDENS(u0, sg, opt=ude.ADAM(0.03))


# d = hls = 2 with one path: most draws leave a hidden layer with no live unit and three zero parameter blocks; this one does not
INPUT_SEED = {(2, 2): 2011}


def _inputs(d, hls):
    """Random x0 and a perturbed Glorot theta, as test_f64_loss_gradient_vs_oracle draws them."""
    rng = np.random.default_rng(INPUT_SEED.get((d, hls), 1000 * d + hls))
    x0 = 0.3 * rng.standard_normal(d)
    theta = bo.init_params(d, hls, seed=3) + 0.05 * rng.standard_normal(sum(bo.num_params(d, hls)))
    return x0, theta


def _set_env(monkeypatch, env):
    for k in ("BSDE_PAIRS", "BSDE_WGRAD", "BSDE_FUSED"):
        monkeypatch.delenv("B200UDE_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("B200UDE_" + k, v)


def _blocks(d, hls):
    """(name, slice) of the parameter blocks in theta order: the u0 net, then [W | b] of each layer of the z net."""
    pu, _ = bo.num_params(d, hls)
    out, o = [("u0net", slice(0, pu))], pu
    for l, (nin, nout) in enumerate(zip((d + 1, hls, hls, hls), (hls, hls, hls, d))):
        out.append((f"z{l}", slice(o, o + nin * nout + nout)))
        o += nin * nout + nout
    return out


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _errors(res, ref, d, hls):
    """res = (loss, grad, u0) of a handle, ref = (loss, grad, u0) of the oracle -> relative errors, per parameter block too."""
    (loss, g, u0), (lo, go, uo) = res, ref
    g = g.cpu().numpy().astype(np.float64)
    e = dict(loss=abs(loss - lo) / abs(lo), u0=abs(u0 - uo) / max(1.0, abs(uo)), grad=_rel(g, go))
    for name, sl in _blocks(d, hls):
        assert np.linalg.norm(go[sl]) > 0, f"the oracle's gradient of block {name} is zero: nothing to compare"
        e[name] = _rel(g[sl], go[sl])
    return e


def _check(tag, e, tol):
    print(f"[{tag}] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    for k, v in e.items():
        t = tol.get(k, tol["grad"])   # the parameter blocks at the gradient's tolerance
        assert v <= t, (tag, k, v, t)


def _same(a, b):
    """Bitwise equality of two (loss, grad, u0) results."""
    return a[0] == b[0] and a[2] == b[2] and torch.equal(a[1], b[1])


def _oracle(theta, d, hls, x0, N, M, seed, **kw):
    t = time.perf_counter()
    ref = bo.loss_and_grad(theta, d, hls, x0, 1.0, N, M, seed, **kw)
    print(f"oracle d={d} hls={hls} N={N} M={M}: {time.perf_counter() - t:.2f} s (numpy fp64, CPU)")
    return ref


# ============================================================================================================================
# 1. The benchmarked configuration (bench.py --config hjb): d = 100, hidden = 110, 20 steps, 10 000 paths, x0 = 0, Flux init
# ============================================================================================================================
BD, BH, BN, BM = 100, 110, 20, 10000


def _bench_solver(ude):
    prob, alg = _problem(ude, BD, BH, np.zeros(BD))
    s = ude.BSDESolver(prob, alg, BN, BM, dtype=torch.float64)
    theta = ude.initial_params_pde(alg)
    s.set_params(theta)
    return s, theta


def _assert_bench_geometry():
    g = geometry(BM, BN, _sm_count())
    _show("bench geometry", g)
    assert min(g.wg_chunks) > WGD       # every k_wgrad CTA refills its ring
    assert g.bwd_rounds > 2             # the persistent k_fused_backward CTAs walk many task groups


def test_bench_config_loss_gradient_and_path_shards_vs_oracle():
    """One iteration at the benchmarked size against the oracle; two uneven path shards (as bench.py's multi-GPU step cuts them)
    add up to the whole batch."""
    _assert_bench_geometry()
    ude = _ude()
    s, theta = _bench_solver(ude)
    res = s.loss_gradient(BM, seed=1)
    ms = s.last_sweep_ms()
    print(f"bench config sweeps: forward {ms[0]:.2f} ms, cotangents {ms[1]:.2f} ms, weight gradients {ms[2]:.2f} ms")
    ref = _oracle(theta, BD, BH, np.zeros(BD), BN, BM, seed=1)
    _check("bench config vs oracle", _errors(res, ref, BD, BH), F64_TOL)
    la, ga, ua = s.loss_gradient(4999, seed=1, path_offset=0, total_paths=BM)
    lb, gb, ub = s.loss_gradient(5001, seed=1, path_offset=4999, total_paths=BM)
    e = dict(loss=abs(la + lb - res[0]) / abs(res[0]), grad=_rel((ga + gb).cpu().numpy(), res[1].cpu().numpy()))
    print(f"[shards 4999 + 5001 vs one call] loss {e['loss']:.2e} grad {e['grad']:.2e}")
    assert ua == ub == res[2]
    assert e["loss"] <= 1e-12 and e["grad"] <= 1e-12   # measured 1.5e-16 and 4.0e-16
    s.close()


def test_bench_config_training_vs_oracle_and_host_loop():
    """train_adam (one direct iteration, then replays of a CUDA graph) against the oracle's ADAM; the host loop loss_gradient +
    adam_step (the update of multi-GPU runs) on a fresh handle runs the same kernels on the same inputs: the same bits."""
    _assert_bench_geometry()
    ude = _ude()
    iters = 3
    s, theta = _bench_solver(ude)
    losses, u0s = s.train_adam(ude.ADAM(0.03), BM, iters, seed0=1)
    losses, u0s, th = losses.cpu().numpy(), u0s.cpu().numpy(), s.get_params()
    s.close()
    t = time.perf_counter()
    th_o, lo, uo = bo.train(theta, BD, BH, np.zeros(BD), 1.0, BN, BM, iters, eta=0.03, seed0=1)
    print(f"oracle: {(time.perf_counter() - t) / iters:.2f} s per ADAM iteration at M = {BM} (numpy fp64, CPU)")
    e = dict(loss=float(np.abs(losses / lo - 1).max()), u0=float((np.abs(u0s - uo) / np.maximum(1.0, np.abs(uo))).max()),
             theta=float(np.abs(th - th_o).max() / np.abs(th_o).max()))
    print(f"[bench config train_adam x{iters} vs oracle] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    # the tolerances of test_f64_adam_history_vs_oracle; measured loss 7.2e-15, theta 1.5e-13 (of max |theta|)
    np.testing.assert_allclose(losses, lo, rtol=1e-7)
    np.testing.assert_allclose(u0s, uo, rtol=1e-7)
    np.testing.assert_allclose(th, th_o, rtol=1e-6, atol=1e-8)

    s, _ = _bench_solver(ude)
    opt = ude.ADAM(0.03)
    hl, hu = [], []
    for i in range(iters):
        loss, g, u0 = s.loss_gradient(BM, seed=1 + i)
        s.adam_step(opt, g)
        hl.append(loss)
        hu.append(u0)
    th_h = s.get_params()
    s.close()
    print(f"[host loop vs train_adam] losses equal {np.array_equal(hl, losses)}, u0s equal {np.array_equal(hu, u0s)}, "
          f"theta max |diff| {np.abs(th_h - th).max():.2e}")
    assert np.array_equal(hl, losses) and np.array_equal(hu, u0s) and np.array_equal(th_h, th)


# ============================================================================================================================
# 2. Kernel variants x shapes
# ============================================================================================================================
SHAPES = [(100, 110, 2001, 13), (110, 110, 77, 5), (110, 111, 41, 3), (2, 2, 1, 1), (9, 16, 8, 4)]


def _assert_shape_geometry(d, hls, M, N):
    """What each shape of SHAPES is there to exercise."""
    sm = _sm_count()
    g = geometry(M, N, sm)
    _show(f"geometry d={d} hls={hls} M={M} N={N}", g)
    if (d, hls) == (100, 110):
        assert min(g.wg_chunks) > WGD                          # the k_wgrad ring wraps in every CTA
        assert g.bwd_rounds >= 3                               # k_fused_backward CTAs walk three task groups
        assert g.bwd_last_group_tasks < FWPC                   # ... and the last group is partial
        assert g.last_tile_paths == 1                          # the last path tile holds one path
        assert g.fwd_last_cta_tiles < FWF and g.fwd2_last_cta_tiles < FP_TILES   # the last forward CTA is partial (both kernels)
    elif (d, hls) == (110, 110):
        assert d % 4 == 2 and d == 110 and hls % 2 == 0        # the largest even widths (fused k_wgrad); a half-used Philox block
    elif (d, hls) == (110, 111):
        assert hls % 2 == 1                                    # the largest fused shape; odd: library weight-gradient GEMMs
    elif (d, hls) == (2, 2):
        assert M == 1 and N == 1 and g.wg_chunks.count(0) == g.wg_splits - 1   # all k_wgrad CTAs but one own no rows
    else:
        assert g.tiles == 1 and g.last_tile_paths == 8 and d % 2 == 1          # exactly one full tile, odd d


_ORACLE = {}
_GRAD_BITS = {}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("d,hls,M,N", SHAPES, ids=[f"d{d}h{h}M{m}N{n}" for d, h, m, n in SHAPES])
def test_variant_vs_oracle(d, hls, M, N, variant, monkeypatch):
    """Every kernel variant on every shape: against the oracle, bit for bit on a repeat; last_sweep_ms() answers exactly when the
    fused sweeps run, which shows the environment reached b200ude_bsde_create."""
    from universal_differential_equations_b200._lib import B200UDEError, EUNSUPPORTED
    _assert_shape_geometry(d, hls, M, N)
    _set_env(monkeypatch, VARIANTS[variant])
    ude = _ude()
    x0, theta = _inputs(d, hls)
    prob, alg = _problem(ude, d, hls, x0)
    s = ude.BSDESolver(prob, alg, N, M, dtype=torch.float64)
    s.set_params(theta)
    r1 = s.loss_gradient(M, seed=11)
    if variant == "fused0":
        with pytest.raises(B200UDEError) as e:
            s.last_sweep_ms()
        assert e.value.code == EUNSUPPORTED
    else:
        assert all(t >= 0 for t in s.last_sweep_ms())
    s.loss_gradient(M, seed=12)
    r2 = s.loss_gradient(M, seed=11)
    s.close()
    assert _same(r1, r2), "not bitwise repeatable"
    if (d, hls) == (100, 110):
        # sums this long end in different last bits in each variant (measured): the environment chose the kernels that ran
        for other, g in _GRAD_BITS.items():
            assert not torch.equal(r1[1], g), f"{variant} gives the bits of {other}"
        _GRAD_BITS[variant] = r1[1]
    key = (d, hls, M, N)
    if key not in _ORACLE:
        _ORACLE[key] = _oracle(theta, d, hls, x0, N, M, seed=11)
    _check(f"{variant} d={d} hls={hls} M={M} N={N}", _errors(r1, _ORACLE[key], d, hls), F64_TOL)


# ============================================================================================================================
# 3. The width limit of the fused sweeps: dim <= 110 and hidden <= 111
# ============================================================================================================================
@pytest.mark.parametrize("d,hls", [(110, 111), (111, 111), (110, 112)])
def test_width_limit_of_the_fused_sweeps(d, hls):
    """At (110, 111) an fp64 handle runs the fused sweeps and a float32 caller gets fp64 arithmetic; one unit more in either width
    and both run on library GEMMs in their own precision.  Both sides against the oracle."""
    from universal_differential_equations_b200._lib import B200UDEError, EUNSUPPORTED
    ude = _ude()
    fused = d <= 110 and hls <= 111
    M, N = 24, 3
    x0, theta = _inputs(d, hls)
    prob, alg = _problem(ude, d, hls, x0)

    s = ude.BSDESolver(prob, alg, N, M, dtype=torch.float64)
    s.set_params(theta)
    res = s.loss_gradient(M, seed=5)
    if fused:
        assert all(t >= 0 for t in s.last_sweep_ms())
    else:
        with pytest.raises(B200UDEError) as e:
            s.last_sweep_ms()
        assert e.value.code == EUNSUPPORTED
    s.close()
    _check(f"fp64 d={d} hls={hls} ({'fused' if fused else 'library'})", _errors(res, _oracle(theta, d, hls, x0, N, M, seed=5), d, hls), F64_TOL)

    s = ude.BSDESolver(prob, alg, N, M, dtype=torch.float32)
    assert s.dtype == (torch.float64 if fused else torch.float32) and s.io_dtype == torch.float32
    th32 = theta.astype(np.float32)
    s.set_params(th32)
    res = s.loss_gradient(M, seed=5)
    s.close()
    x32 = x0.astype(np.float32).astype(np.float64) if not fused else x0   # an fp32 handle holds x0 in float32
    ref = _oracle(th32.astype(np.float64), d, hls, x32, N, M, seed=5)
    # fp64 arithmetic, results rounded to float32: the tolerances of test_f32_caller_gets_double_arithmetic_by_default (measured loss
    # 1.8e-16, gradient 2.5e-8); past the limit fp32 library GEMMs (measured up to 1.8e-8, 1.7e-7)
    tol = dict(loss=1e-9, grad=2e-7) if fused else F32_TOL
    e = _errors(res, ref, d, hls)
    _check(f"float32 caller d={d} hls={hls} ({'fp64 fused' if fused else 'fp32 library'})", {k: e[k] for k in ("loss", "grad")}, tol)


# ============================================================================================================================
# 4. Changing n_paths on one handle
# ============================================================================================================================
def test_changing_n_paths_on_one_handle():
    """prepare() lays out the constant rows of the tapes ([t; 1] of the inputs, the ones rows of the hidden layers) for the number of
    paths of the call: 10 000, then 37, then 10 000 paths again on one handle."""
    ude = _ude()
    d, hls, N, cap = 100, 110, 20, 10000
    x0, theta = _inputs(d, hls)
    prob, alg = _problem(ude, d, hls, x0)
    s = ude.BSDESolver(prob, alg, N, cap, dtype=torch.float64)
    s.set_params(theta)
    r1 = s.loss_gradient(cap, seed=21)
    r2 = s.loss_gradient(37, seed=22)
    r3 = s.loss_gradient(cap, seed=21)
    s.close()
    print(f"[10000 -> 37 -> 10000 paths] third call bitwise equal to the first: {_same(r1, r3)}")
    assert _same(r1, r3)
    _check("37 paths after 10000 vs oracle", _errors(r2, _oracle(theta, d, hls, x0, N, 37, seed=22), d, hls), F64_TOL)
