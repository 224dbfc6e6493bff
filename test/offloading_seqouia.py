# CUDA_VISIBLE_DEVICES=0,1 OMP_NUM_THREADS=48 torchrun --nproc_per_node=2 test/offloading_seqouia.py --budget 12288 --prefill 130048 --dataset demo --target llama-7B-128K --on_chip 9 --seed 1
"""The reference's Sequoia-tree entry point (same flags and report lines) on the GPU-native engine — see
`triforce_b200.cli.run_offloading_seqouia`."""
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from triforce_b200.cli import run_offloading_seqouia  # noqa: E402

if __name__ == "__main__":
    run_offloading_seqouia()
