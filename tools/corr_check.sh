#!/bin/bash
cd "$(dirname "$0")/.."
timeout 200 python -m pytest tests/test_linalg.py -m gpu -x -q 2>&1 | tail -2
timeout 200 python tools/bench_ops.py --ops correlate 2>&1 | tail -3 | cut -c1-110
