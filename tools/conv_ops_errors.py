"""Normwise errors rho = ||got - ref||_2 / ||ref||_2 of every GEMM output of the image-convolution cases of
tests/test_conv_ops_table.py on the GPU, one JSON line per (case, output), with the GPU name and power limit.

    python tools/conv_ops_errors.py OUT.jsonl"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import test_gpu_conv_ops as T  # noqa: E402
from test_conv_ops_table import CONV_CASES, tau_of  # noqa: E402


def gpu_name():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main(path):
    gpu, day = gpu_name(), time.strftime("%Y-%m-%d")
    with open(path, "w") as f:
        for c in CONV_CASES:
            try:
                T.run_case(c)
            except AssertionError as e:          # still report the measured errors
                print(c["id"], "failed:", str(e)[:300])
            for k in ("z", "dx", "dw"):
                if (c["id"], k) not in T.RHO:
                    continue
                f.write(json.dumps({"case": c["id"], "lib": c["lib"], "output": k, "rho": T.RHO[(c["id"], k)],
                                    "tau": tau_of(c, k), "gpu": gpu, "time": day}) + "\n")
    print(open(path).read())


if __name__ == "__main__":
    main(sys.argv[1])
