"""The CTA-width sweep of otb_sample_step's kernel (DESIGN.md 4.11): builds tools/sample_step_sweep.cu, which compiles the
library's sample_step_kernel at 32 (one warp per row), 64, 128, 256 and 512 threads per row, into a temporary directory and
runs it.  It prints one JSON object: the card, its power limit and maximum SM clock read in the same run, and per
(rows, V, width) the median, min and max microseconds per launch over --reps windows of 60 launches, with whether the
drawn tokens equal the 256-thread launch's.  Needs a GPU.

    python tools/sample_step_sweep.py [--reps 21]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from ctc_model import card  # noqa: E402
from opentransformer_b200 import build  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=21)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, 'sample_step_sweep')
        subprocess.run([build._nvcc()] + build.NVCC_FLAGS[:5] + ['-o', exe, os.path.join(HERE, 'sample_step_sweep.cu')],
                       check=True, capture_output=True, text=True)
        rows = json.loads(subprocess.run([exe, str(args.reps)], check=True, capture_output=True, text=True).stdout)
    print(json.dumps({'card': card(), 'reps': args.reps, 'launches_per_window': 60, 'results': rows}))


if __name__ == '__main__':
    main()
