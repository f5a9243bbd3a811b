"""Write tests/golden/operator_bits.json: for every case of tests/operator_bits_cases.py, the sha256 of the bits of out, status,
the loss, grad_theta and grad_u0 that the operator UDE kernels give (needs a GPU).

    python tools/make_golden_operator_bits.py

The file was written by the library before the operator kernels were rewritten over shared helpers (one RKC2 recurrence, one
adaptive step loop, one replay of the accepted steps); tests/test_gpu_operator_bits.py checks that the library still gives
those bits.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import operator_bits_cases as C  # noqa: E402


def main():
    digests = {}
    for case in C.CASES:
        r = C.run(*case)
        digests[C.key(*case)] = C.bits_digest(*r)
        print(C.key(*case), "status", sorted(set(r[1].tolist())), "loss", float(r[2][0]), "|grad_theta|", float(abs(r[3]).sum()), flush=True)
    with open(C.GOLDEN, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{C.GOLDEN}: {len(digests)} cases")


if __name__ == "__main__":
    main()
