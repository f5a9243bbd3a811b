"""b200ude_create's answer for every descriptor of the grid in descriptor_grid.py: which descriptors pass validation, and the
return code and message of each refusal, against tests/golden/descriptor_outcomes.npz (tools/make_golden_descriptors.py).
Validation runs before the device probe, so the test runs with and without a GPU; on a GPU a descriptor that passes validation
must also get its handle (B200UDE_OK), or B200UDE_ENODEVICE on a device that is not sm_90."""
import os

import numpy as np

import descriptor_grid as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_descriptor_gets_its_recorded_answer():
    from universal_differential_equations_b200 import _lib
    want = np.load(os.path.join(ROOT, "tests", "golden", "descriptor_outcomes.npz"))
    keys, rcs, msgs = G.outcomes(_lib)
    assert G.key_digest(keys) == str(want["key_digest"]), "the grid changed: regenerate the golden file at the commit that defines the answers"
    messages = [str(m) for m in want["messages"]]
    expected = [(int(r), messages[i]) for r, i in zip(want["rc"], want["msg_index"])]
    bad = [(k, e, (r, m)) for k, e, r, m in zip(keys, expected, rcs, msgs) if e != (r, m)]
    assert not bad, f"{len(bad)} of {len(keys)} descriptors answered differently (key, recorded, now), e.g. {bad[:5]}"
    assert (want["rc"] == 0).any() and (want["rc"] != 0).any()
