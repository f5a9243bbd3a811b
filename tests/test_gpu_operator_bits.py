"""Every operator UDE kernel, in fp32 and fp64, bit for bit against out, status, the loss, grad_theta and grad_u0 recorded
before the kernels were rewritten over shared helpers (tests/golden/operator_bits.json, cases in operator_bits_cases.py): the
rewrite moved code, not arithmetic, so not one bit may change."""
import json

import numpy as np
import pytest

pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import operator_bits_cases as C  # noqa: E402


@pytest.mark.parametrize("case", C.CASES, ids=[C.key(*c) for c in C.CASES])
def test_recorded_bits(case):
    out, status, loss, g, gu = C.run(*case)
    with open(C.GOLDEN) as f:
        recorded = json.load(f)[C.key(*case)]
    if case[5] == "max_steps":   # a failed trajectory's unreached saves are NaN
        assert (status == 2).any() and set(status.tolist()) <= {0, 2} and np.isnan(out[-1][:, status == 2]).all()
    else:
        assert (status == 0).all() and np.isfinite(out).all() and np.isfinite(g).all()
    assert C.bits_digest(out, status, loss, g, gu) == recorded, "out, status, loss, grad_theta or grad_u0 differ from the recorded bits"


@pytest.mark.parametrize("dtype", C.DTYPES)
def test_cases_reach_their_branches(dtype):
    """The stage-cap cases step at the cap's h = beta(3) / (1.05 eigen_est): they need at least span / h accepted steps and
    succeed with two more, which error control alone would not give.  Some adaptive case covers its 10 save intervals in
    fewer accepted steps, so save times fall inside steps."""
    import math

    from universal_differential_equations_b200.sciml import _rkc2_beta
    span = 0.04 * 10
    for case in [c for c in C.CASES if c[5] == "stage_cap" and c[6] == dtype]:
        n = math.ceil(span / (_rkc2_beta(3) / (1.05 * 2000.0)))
        assert (C.status_at(case, n - 1) == 2).all() and (C.status_at(case, n + 2) == 0).all(), case
    free = [c for c in C.CASES if c[0].endswith("_adaptive") and c[5] == "" and c[6] == dtype]
    assert any((C.status_at(c, 9) == 0).all() for c in free)
