#!/usr/bin/env python
"""A handful of tf_verify_attn launches at one shape, for a profiler to count DRAM bytes on (bench.py runs this under
`ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum` after its timed region to fill `roofline.traffic`).
    python tools/attn_traffic_probe.py --kv_len 124935 --rows 7 --heads 32 [--head_dim 128] [--launches 4]"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from triforce_b200 import ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv_len", type=int, required=True)
    ap.add_argument("--rows", type=int, required=True)
    ap.add_argument("--heads", type=int, required=True)
    ap.add_argument("--head_dim", type=int, default=128)
    ap.add_argument("--launches", type=int, default=4)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    S, R, H, d = args.kv_len, args.rows, args.heads, args.head_dim
    L = 2  # alternate two layers so that no launch finds its keys in the 50 MB L2
    Ks = torch.randn((L, H, S + 64, d), device=dev, dtype=torch.float16)
    Vs = torch.randn((L, H, S + 64, d), device=dev, dtype=torch.float16)
    q = torch.randn((R, H, d), device=dev, dtype=torch.float16)
    o = torch.empty_like(q)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, dev)
    for i in range(args.launches):
        ops.verify_attn(q, maps, i % L, S, R, H, d, 0.08837890625 if d == 128 else 0.125, o, ws)
    torch.cuda.synchronize()
    print("probe done")


if __name__ == "__main__":
    main()
