#!/usr/bin/env python
"""Record the output digests of tests/test_gpu_gemm_persistent.py's cases with the r3g library of another tree (the
commit before a GEMM change, extracted with `git archive <commit> | tar -x -C ab_parent` and built there):
  python tools/make_gemm_golden.py --tree ab_parent --out tests/golden/gemm_persistent.json"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", required=True, help="repository tree whose built libr3g computes the digests")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(os.path.abspath(args.tree), "3d-re-gen_b200"))
    import r3g
    import test_gpu_gemm_persistent as T
    print("r3g from", os.path.dirname(r3g.__file__))
    golden = {name: T.digest(fn()) for name, fn in T.cases().items()}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(golden, f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(golden), "digests ->", args.out)


if __name__ == "__main__":
    main()
