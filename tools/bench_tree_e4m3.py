"""The Sequoia tree path over an E4M3 full-KV store and E4M3 weights, measured on one GPU.

    python tools/bench_tree_e4m3.py                 # kernel lines, then the four workload legs (one subprocess each)
    python tools/bench_tree_e4m3.py --kernel-only
    python tools/bench_tree_e4m3.py --leg e4m3,e4m3,130048

Kernel: tf_tree_attn_tc_e4m3 against tf_tree_attn_tc over the dequantized store D, alternated in one process (CUDA events,
median of 5 rounds of 10 launches), R = 512 rows with the real 512-node tree mask, d = 128, one layer of 40 (MHA) or 32 query /
8 KV heads, at kv_len 49 664 and 130 560.  Outputs are asserted bit-identical at every timed size.  FLOP = 4 R kv_len H d.

Workload: BASELINE cfg5's geometry (Llama2-13B shape, 40 layers, budget 8192, the 512-node tree, SingleGpuLlama) with seeded random-init
weights (not acceptance-calibrated, so tokens per round say little about a real model).  Per leg: prefill time, ms per tree
round (growth + verify, shown separately, median over the timed rounds), tokens per round and peak device memory.  Every leg
draws its fp16 weights on the GPU and keeps them in host memory, so the state dict is never resident beside the model."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from triforce_b200 import ops  # noqa: E402

DEV = "cuda"
PEAK_TFLOPS = 989.0  # H100 SXM dense fp16 data-sheet figure (700 W card)
LEGS = [("fp16", "fp16", 49152), ("e4m3", "fp16", 49152), ("e4m3", "e4m3", 49152), ("e4m3", "e4m3", 130048)]


def gpu_info() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # the numbers still stand; say that the card could not be read
        return f"nvidia-smi unavailable ({e!r})"


def _dequant(codes, e):
    return (codes.view(torch.float8_e4m3fn).double() * torch.exp2(e.double()).unsqueeze(-1)).half()


def _store(H, cap, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    parts = []
    for _ in range(2):
        c = torch.randint(0, 256, (1, H, cap, 128), generator=g, device=DEV, dtype=torch.uint8)
        c = torch.where((c & 0x7F) == 0x7F, c ^ 1, c)
        e = torch.randint(-12, 2, (1, H, cap), generator=g, device=DEV, dtype=torch.int8)
        parts.append((c.contiguous(), e.contiguous()))
    (kc, ke), (vc, ve) = parts
    return ops.E4m3Store(kc, vc, ke, ve), _dequant(kc, ke), _dequant(vc, ve)


def kernel_lines():
    from triforce_b200.spectree import load_grow_map, pack_mask_bits

    R, d = 512, 128
    mask = pack_mask_bits(load_grow_map("512")["mask"]).to(DEV)
    for Hq, Hkv in ((40, 40), (32, 8)):
        for kv_len in (49664, 130560):
            st, KD, VD = _store(Hkv, kv_len, kv_len + Hkv)
            maps = ops.KVTensorMaps(KD, VD)
            q = (torch.randn((R, Hq, d), device=DEV) * 0.05).half()
            ws = ops.tree_attn_tc_workspace(R, Hq, kv_len, DEV)
            o8, o16 = torch.empty_like(q), torch.empty_like(q)
            scale = d ** -0.5

            def e4m3():
                ops.tree_attn_tc_e4m3(q, st, 0, kv_len, R, Hq, Hkv, d, scale, mask, R, o8, ws)

            def fp16():
                if Hq == Hkv:
                    ops.tree_attn_tc(q, maps, 0, kv_len, R, Hq, d, scale, mask, R, o16, ws)
                else:
                    ops.tree_attn_tc_gqa(q, maps, 0, kv_len, R, Hq, Hkv, d, scale, mask, R, o16, ws)

            times = {"e4m3": [], "fp16": []}
            for fn in (e4m3, fp16):
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            for _ in range(5):
                for name, fn in (("e4m3", e4m3), ("fp16", fp16)):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(10):
                        fn()
                    b.record()
                    b.synchronize()
                    times[name].append(a.elapsed_time(b) / 10)
            e4m3()
            fp16()
            torch.cuda.synchronize()
            assert torch.equal(o8, o16), f"outputs differ at Hq={Hq} Hkv={Hkv} kv_len={kv_len}"
            flop = 4.0 * R * kv_len * Hq * d
            line = {"kernel": "tree_attn_tc", "R": R, "Hq": Hq, "Hkv": Hkv, "kv_len": kv_len, "bit_identical": True}
            for name in ("fp16", "e4m3"):
                ms = statistics.median(times[name])
                tf = flop / ms / 1e9
                line[name] = {"ms": round(ms, 4), "tflops": round(tf, 1), "share_of_989": round(tf / PEAK_TFLOPS, 3)}
            line["e4m3_over_fp16"] = round(line["e4m3"]["ms"] / line["fp16"]["ms"], 3)
            print(json.dumps(line), flush=True)
            del st, KD, VD, maps
            torch.cuda.empty_cache()


@torch.inference_mode()
def run_leg(kv: str, weights: str, P: int, rounds: int = 4):
    from triforce_b200.config import named_config
    from triforce_b200.rng import CounterNoise
    from triforce_b200.spectree import SpecTree, load_grow_map
    from triforce_b200.synth import cuda_state_dict, numpy_prompt
    from triforce_b200.tp import SingleGpuLlama

    cfg = named_config("llama-13B-128K")
    gm = load_grow_map("512")
    gen_len = (rounds + 1) * 24 + 64
    llm = SingleGpuLlama("llama-13B-128K", local_rank=0, world_size=1, prefill=P, gen_len=gen_len, retrieval_budget=8192,
                         retrieval_chunk_size=8, temperature=0.6, top_p=0.9, config=cfg, tree_size=gm["size"], kv_dtype=kv,
                         weight_dtype=weights)
    llm.init_parameters(state_dict=cuda_state_dict(cfg, seed=1, device=DEV, host=True), cuda_graphs=False)
    st = SpecTree(engine=llm, temperature=0.6, top_p=0.9, max_length=P + gen_len, grow_map=gm, vocab_size=cfg.vocab_size,
                  noise=CounterNoise(3, device=DEV))
    ids = numpy_prompt(P, seed=5)[0].to(DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    nt = st.prefill(prefix=ids)
    torch.cuda.synchronize()
    prefill_s = time.perf_counter() - t0
    grow, verify, counts = [], [], []
    for r in range(rounds + 1):  # round 0 warms up
        t0 = time.perf_counter()
        st.construct_grow_map(next_token=nt)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        nt, acc, _ = st.verify()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if r:
            grow.append((t1 - t0) * 1e3)
            verify.append((t2 - t1) * 1e3)
            counts.append(acc)
        if nt is None:
            break
        nt = nt.unsqueeze(0)
    g, v = statistics.median(grow), statistics.median(verify)
    print(json.dumps({"leg": {"kv_dtype": kv, "weight_dtype": weights, "prefill": P}, "weights": "random-init (seed 1)",
                      "prefill_s": round(prefill_s, 2), "ms_per_round": round(g + v, 1), "growth_ms": round(g, 1),
                      "verify_ms": round(v, 1), "tokens_per_round": counts, "rounds_timed": len(counts),
                      "peak_device_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                      "device_used_gb": round((lambda f, t: (t - f) / 1e9)(*torch.cuda.mem_get_info()), 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel-only", action="store_true")
    ap.add_argument("--leg", type=str, default=None, help="kv_dtype,weight_dtype,prefill: run one workload leg in this process")
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tree_e4m3 needs a GPU")
    if args.leg:
        kv, w, P = args.leg.split(",")
        run_leg(kv, w, int(P), args.rounds)
        return
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    kernel_lines()
    if args.kernel_only:
        return
    for kv, w, P in LEGS:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", f"{kv},{w},{P}", "--rounds", str(args.rounds)],
                           capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        if r.returncode != 0 or not lines:
            print(json.dumps({"leg": {"kv_dtype": kv, "weight_dtype": w, "prefill": P}, "error": r.returncode,
                              "tail": (r.stdout + r.stderr)[-1500:]}), flush=True)
        else:
            print(lines[-1], flush=True)
    print(json.dumps({"gpu": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
