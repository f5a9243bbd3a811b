"""Write tests/golden/descriptor_outcomes.npz: what b200ude_create answers for every descriptor of tests/descriptor_grid.py.

Run with the library built (no GPU needed):  python tools/make_golden_descriptors.py
tests/test_descriptor_outcomes.py checks the library against the file, so that a change of the host layer that moves a refusal,
its message, or which descriptors pass validation shows up as a test failure.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import descriptor_grid as G  # noqa: E402
from universal_differential_equations_b200 import _lib  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "descriptor_outcomes.npz")


def main():
    keys, rcs, msgs = G.outcomes(_lib)
    messages = sorted(set(msgs))   # "" (passes validation) first
    np.savez_compressed(OUT, key_digest=np.array(G.key_digest(keys)), rc=np.array(rcs, dtype=np.int8),
                        msg_index=np.array([messages.index(m) for m in msgs], dtype=np.int16), messages=np.array(messages))
    valid = sum(rc == 0 for rc in rcs)
    print(f"{OUT}: {len(keys)} descriptors, {valid} pass validation, {len(messages) - 1} distinct refusals")


if __name__ == "__main__":
    main()
