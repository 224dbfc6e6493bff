# CUDA_VISIBLE_DEVICES=0 python test/on_chip.py --prefill 124928 --budget 4096 --chunk_size 8 --top_p 0.9 --temp 0.6 --gamma 6 --dataset 128k
"""The reference's on-chip entry point (same flags and report lines) on the GPU-native engine — see
`triforce_b200.cli.run_on_chip`."""
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from triforce_b200.cli import run_on_chip  # noqa: E402

if __name__ == "__main__":
    run_on_chip()
