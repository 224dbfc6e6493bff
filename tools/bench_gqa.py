"""Grouped-query targets on the GPU: the llama-7B-gqa8-128K workload, and its full-KV verify attention against the MHA
launch at the same key count, in one command.

Workload leg: llama-7B-gqa8-128K (32 query / 8 KV heads, synthetic random-init fp16 weights) with the Llama-68M draft,
prefill 124 928, budget 4096, chunk 8, gamma 6, T 0.6, top_p 0.9, run as bench.py runs cfg2: the autoregressive baseline
(full-KV decode step as one CUDA graph + fused sampling, CUDA events over --ar-steps steps) and TriForce through the
whole-loop device graph (DeviceLoopRun, CUDA events over --steps outer steps after --warmup).  Reports tokens/s, ms per
outer step, AR ms/token and peak device memory.

Kernel leg: times tf_verify_attn_gqa (8 token rows, 32 query / 8 KV heads, d = 128) and tf_verify_attn (8 rows, 32 MHA heads: the
llama-7B-128K shape) over 124 944 keys of one layer, alternating the two in rounds, with CUDA events around many
launches.  Prints the time per launch, the algorithmic bytes (kv_len · heads · d · 2 (K+V) · 2 B) over that time, the
share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and the GPU's name and power limit read in the same run.

    python tools/bench_gqa.py [--steps 8] [--warmup 2] [--kv-len 124944] [--launches 200] [--rounds 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from triforce_b200 import ops  # noqa: E402
from triforce_b200.rope import softmax_scale  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_identity() -> dict:
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:  # the number is reported as missing, never guessed
        out["power_limit_error"] = repr(e)
    return out


def workload(a) -> dict:
    """The llama-7B-gqa8-128K TriForce workload through the whole-loop device graph (see the module docstring)."""
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from triforce_b200.config import named_config
    from triforce_b200.decoding import _sample_token
    from triforce_b200.device_loop import DeviceLoopRun
    from triforce_b200.engine import GraphInferenceEngine
    from triforce_b200.llama import LlamaModel
    from triforce_b200.rng import TorchNoise
    from triforce_b200.sampling import norm_logits
    from triforce_b200.synth import cuda_state_dict

    dev = torch.device("cuda", 0)
    torch.manual_seed(a.seed)
    P, B, chunk, gamma, temp, top_p = a.prefill, 4096, 8, 6, 0.6, 0.9
    cfg_t, cfg_d = named_config("llama-7B-gqa8-128K"), named_config("llama-68M")
    target = LlamaModel(cfg_t, cuda_state_dict(cfg_t, seed=1, device=dev), device=dev)
    draft = LlamaModel(cfg_d, cuda_state_dict(cfg_d, seed=2, device=dev), device=dev, is_draft=True)
    torch.cuda.empty_cache()
    cache = FlashSimpleCache(target, P + a.gen_len + 16)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=gamma, chunk_size=chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.engine.target_prefill_chunk = 1024
    ge.initialize_cuda_graph(gamma, probs=True, temperature=temp, top_p=top_p)
    g = torch.Generator().manual_seed(a.seed)
    input_ids = torch.randint(0, cfg_t.vocab_size, (1, P), generator=g).to(dev)
    tok = type("Tok", (), {"eos_token_id": 2, "decode": lambda self, *x, **k: ""})()
    noise = TorchNoise(dev)
    with torch.inference_mode():
        t0 = time.time()
        logits = ge.inference(input_ids=input_ids)
        torch.cuda.synchronize()
        prefill_s = time.time() - t0
        expo = torch.empty(cfg_t.vocab_size, dtype=torch.float32, device=dev)
        nxt = _sample_token(norm_logits(logits[:, -1, :], temperature=temp, top_k=-1, top_p=top_p), noise, expo)

        def ar_step(tk):
            lg = ge.decode_step(tk)
            return _sample_token(norm_logits(lg[:, -1, :], temperature=temp, top_k=-1, top_p=top_p), noise, expo)

        for _ in range(3):
            nxt = ar_step(nxt)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.ar_steps):
            nxt = ar_step(nxt)
        e1.record()
        torch.cuda.synchronize()
        ar_ms = e0.elapsed_time(e1) / a.ar_steps
        run = DeviceLoopRun(tok, ge, gamma=gamma, top_p=top_p, temperature=temp, seed=a.seed, max_new=a.gen_len)
        run.prefill(input_ids, skip_target_prefill=True)
        for _ in range(a.warmup):
            run.step()
        torch.cuda.synchronize()
        n0, acc0, dr0 = run.n, run.accepted_count, run.draft_count
        e0.record()
        for _ in range(a.steps):
            run.step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        tokens = run.n - n0
    out = {"workload": f"llama-7B-gqa8-128K (random-init fp16 std 0.02) + llama-68M draft, prefill {P}, budget {B}, chunk {chunk}, "
                       f"gamma {gamma}, T {temp}, top_p {top_p}; TriForce through the whole-loop device graph",
           "tokens_per_s": tokens / (ms * 1e-3), "ms_per_step": ms / a.steps, "tokens_per_step": tokens / a.steps, "steps": a.steps,
           "warmup": a.warmup, "acceptance_rate": (run.accepted_count - acc0) / max(run.draft_count - dr0, 1),
           "ar_ms_per_token": ar_ms, "ar_tokens_per_s": 1000.0 / ar_ms, "ar_steps": a.ar_steps,
           "prefill_seconds": prefill_s, "peak_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9}
    del run, ge, target, draft, cache, graph_cache, draft_cache
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv-len", type=int, default=124944)
    ap.add_argument("--rows", type=int, default=8)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--steps", type=int, default=8, help="timed TriForce outer steps of the workload leg")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ar-steps", dest="ar_steps", type=int, default=24)
    ap.add_argument("--prefill", type=int, default=124928)
    ap.add_argument("--gen-len", dest="gen_len", type=int, default=1024, help="KV capacity reserved for generated tokens")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gqa: no CUDA device (this script measures the GPU only)")
    d, Hq, Hkv, Hmha, R, kv_len = 128, 32, 8, 32, a.rows, a.kv_len
    cap = (kv_len + 1023) // 1024 * 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    scale = softmax_scale(d)
    legs = {}
    for name, H, nq in (("gqa_32q_8kv", Hkv, Hq), ("mha_32", Hmha, Hmha)):
        K = torch.randn((1, H, cap, d), generator=g, device="cuda").half()
        V = torch.randn((1, H, cap, d), generator=g, device="cuda").half()
        q = torch.randn((R, nq, d), generator=g, device="cuda").half()
        maps = ops.KVTensorMaps(K, V)
        out = torch.empty_like(q)
        if name.startswith("gqa"):
            ws = ops.verify_attn_gqa_workspace(nq, H, d, "cuda")
            fn = lambda q=q, maps=maps, out=out, ws=ws, nq=nq, H=H: ops.verify_attn_gqa(q, maps, 0, kv_len, R, nq, H, d, scale, out, ws)
        else:
            ws = ops.verify_attn_workspace(ops.VERIFY_MAX_ROWS, H, d, "cuda")
            fn = lambda q=q, maps=maps, out=out, ws=ws, H=H: ops.verify_attn(q, maps, 0, kv_len, R, H, d, scale, out, ws)
        legs[name] = {"fn": fn, "bytes": kv_len * H * d * 2 * 2, "keep": (K, V, q, out, ws), "ms": []}
    for leg in legs.values():  # warm-up: module load, attributes, L2 state
        for _ in range(20):
            leg["fn"]()
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for leg in legs.values():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                leg["fn"]()
            e1.record()
            torch.cuda.synchronize()
            leg["ms"].append(e0.elapsed_time(e1) / a.launches)
    res = {"gpu": gpu_identity(), "kv_len": kv_len, "rows": R, "launches_per_round": a.launches, "rounds": a.rounds}
    for name, leg in legs.items():
        ms = sorted(leg["ms"])[len(leg["ms"]) // 2]
        res[name] = {"ms_per_launch_median": ms, "ms_per_launch_all": leg["ms"], "algorithmic_bytes": leg["bytes"],
                     "tb_per_s": leg["bytes"] / (ms * 1e-3) / 1e12, "share_of_3_35_tb_s": leg["bytes"] / (ms * 1e-3) / HBM_BYTES_PER_S}
    res["gqa_over_mha_time"] = res["gqa_32q_8kv"]["ms_per_launch_median"] / res["mha_32"]["ms_per_launch_median"]
    legs.clear()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    res["workload_llama_7B_gqa8_128K"] = workload(a)
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
