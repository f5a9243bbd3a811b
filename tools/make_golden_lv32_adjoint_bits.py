"""Write tests/golden/lv32_wm_adjoint_bits.json: for every case of tests/lv32_shared_points.py, the sha256 of the bits of out, the
loss and grad_u0 that the warp-collective LV 2-32-32-2 forward and interpolating adjoint give (needs a GPU).

    python tools/make_golden_lv32_adjoint_bits.py

The file was written by the library before the adjoint evaluated the shared step points once (stage 5 of a step and stage 0 of
the step below at the same state); tests/test_gpu_lv32_shared_points.py checks that the library still gives those bits.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lv32_shared_points as C  # noqa: E402


def main():
    os.environ["B200UDE_FWD_WM"] = "1"
    os.environ["B200UDE_ADJ_WM"] = "1"
    digests = {}
    for case in C.CASES:
        out, loss, _, gu = C.run(*case)
        digests[C.key(*case)] = C.bits_digest(out, loss, gu)
    with open(C.GOLDEN, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{C.GOLDEN}: {len(digests)} cases")


if __name__ == "__main__":
    main()
