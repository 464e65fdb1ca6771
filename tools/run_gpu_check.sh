# Dev helper: the GPU tests and timings to re-run on an H100 after a kernel change.
set -x
timeout 1500 python -m pytest tests -m gpu -q 2>&1 | tail -5
timeout 300 python tools/unprofiled_time.py            # c2 / c4 / c3, device time of the async C-ABI
timeout 300 python tools/quick_time.py --bf16 c3 2>&1 | grep "loss+grad"
timeout 300 python tools/joint_time.py 2>&1 | tail -3
