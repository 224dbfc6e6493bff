"""E4M3 projection weights against fp16, in one command:

1. per-projection launches at the 7B shapes (q|k|v 12288x4096, o 4096x4096, gate|up 22016x4096 with SiLU, down 4096x11008,
   lm_head 32000x4096 with the fp32 epilogue), M = 1, 8 and 17 rows (one, two and three token blocks): tf_stream_linear on the
   fp16 matrix D against tf_stream_linear_e4m3 on its codes, alternated in the same run and timed with CUDA events over many
   launches.  The outputs of the timed sizes are asserted bit-identical before timing;
2. all projections of one 8-row 7B verify forward (32 layers x 4 projections + lm_head) captured as one CUDA graph, fp16
   against e4m3, alternated;
3. the cfg2 workload (llama-7B-128K with random-init weights + llama-68M draft, prefill 124 928, budget 4096, chunk 8, gamma 6,
   TriForce through the whole-loop device graph) with fp16 weights / fp16 KV, e4m3 weights / fp16 KV and e4m3 weights / e4m3 KV,
   each in a subprocess of its own: tokens/s, ms per outer step, autoregressive ms/token, prefill seconds, peak device memory.

Prints one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/bench_weights_e4m3.py [--iters 200] [--rounds 5] [--steps 8] [--no-workload]

Bandwidth is algorithmic bytes over time: N·K·2 for fp16, N·K + N (codes and exponents) for e4m3.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from triforce_b200 import ops  # noqa: E402

SHAPES = {"qkv": (12288, 4096, 0), "o": (4096, 4096, 0), "gate_up": (22016, 4096, 1), "down": (4096, 11008, 0),
          "lm_head": (32000, 4096, 2)}


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        pl, sm = out.strip().split(",")[:2]
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(pl), float(sm)
    except Exception as e:  # the numbers still stand; say why the limit is missing
        info["power_limit_error"] = repr(e)
    return info


def workload(a) -> dict:
    """The cfg2 TriForce workload with `a.weights` projection weights on an `a.kv` full-KV store (see the module docstring)."""
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
    cfg_t, cfg_d = named_config("llama-7B-128K"), named_config("llama-68M")
    sd = cuda_state_dict(cfg_t, seed=1, device=dev)
    target = LlamaModel(cfg_t, sd, device=dev, weight_dtype=a.weights)
    del sd
    draft = LlamaModel(cfg_d, cuda_state_dict(cfg_d, seed=2, device=dev), device=dev, is_draft=True)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    cache = FlashSimpleCache(target, P + a.gen_len + 16, kv_dtype=a.kv)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=gamma, chunk_size=chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
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
        n0 = run.n
        e0.record()
        for _ in range(a.steps):
            run.step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        tokens = run.n - n0
    return {"weight_dtype": a.weights, "kv_dtype": a.kv, "tokens_per_s": tokens / (ms * 1e-3), "ms_per_step": ms / a.steps,
            "tokens_per_step": tokens / a.steps, "steps": a.steps, "ar_ms_per_token": ar_ms, "prefill_seconds": prefill_s,
            "peak_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9}


def alternate(fns: dict, iters: int, rounds: int) -> dict:
    for f in fns.values():
        for _ in range(20):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(rounds):  # alternate the variants, one timed window each per round
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters)
    return times


def median(xs):
    return sorted(xs)[len(xs) // 2]


def launches(args) -> dict:
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(args.seed)
    ws = ops.stream_linear_workspace(dev)
    out = {}
    for name, (N, K, epi) in SHAPES.items():
        W = (torch.randn((N, K), generator=g, device=dev) * 0.02).half()
        m8 = ops.E4m3WeightMap.quantize(W, silu=epi == 1)
        D = ops.weight_dequantize_e4m3(m8.codes, m8.exps)
        del W
        m16 = ops.WeightMap(D, silu=epi == 1)
        row = {}
        for M in (1, 8, 17):
            x = torch.randn((M, K), generator=g, device=dev).half()
            n_out = N // 2 if epi == 1 else N
            dt = torch.float32 if epi == 2 else torch.float16
            y16 = torch.empty((M, n_out), dtype=dt, device=dev)
            y8 = torch.empty_like(y16)
            kw = dict(silu=epi == 1, out_fp32=epi == 2, workspace=ws)
            f16 = lambda x=x, y=y16, kw=kw: ops.stream_linear(x, m16, out=y, **kw)
            f8 = lambda x=x, y=y8, kw=kw: ops.stream_linear(x, m8, out=y, **kw)
            f16()
            f8()
            torch.cuda.synchronize()
            assert torch.equal(y16, y8), f"{name} M={M}: tf_stream_linear_e4m3 differs from tf_stream_linear on D"
            t = alternate({"fp16": f16, "e4m3": f8}, args.iters, args.rounds)
            b16, b8 = N * K * 2, N * K + N
            ms16, ms8 = median(t["fp16"]), median(t["e4m3"])
            row[f"M{M}"] = {"fp16_us": round(ms16 * 1e3, 2), "e4m3_us": round(ms8 * 1e3, 2),
                            "fp16_TBps": round(b16 / ms16 / 1e9, 3), "e4m3_TBps": round(b8 / ms8 / 1e9, 3),
                            "e4m3_over_fp16": round(ms8 / ms16, 3), "bit_identical": True,
                            "fp16_us_all": [round(v * 1e3, 2) for v in t["fp16"]], "e4m3_us_all": [round(v * 1e3, 2) for v in t["e4m3"]]}
        out[name] = row
        del m8, m16, D
        torch.cuda.empty_cache()
    return out


def forward_graph(args) -> dict:
    """All projections of one 8-row verify forward of the 7B target, as one CUDA graph (PDL between the launches)."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(args.seed + 1)
    ws = ops.stream_linear_workspace(dev)
    M, L = 8, 32
    layers16, layers8 = [], []
    for _ in range(L):
        l16, l8 = [], []
        for name in ("qkv", "o", "gate_up", "down"):
            N, K, epi = SHAPES[name]
            W = (torch.randn((N, K), generator=g, device=dev) * 0.02).half()
            l16.append(ops.WeightMap(W, silu=epi == 1))
            l8.append(ops.E4m3WeightMap.quantize(W, silu=epi == 1))
        layers16.append(l16)
        layers8.append(l8)
    Wh = (torch.randn((32000, 4096), generator=g, device=dev) * 0.02).half()
    heads = {"fp16": ops.WeightMap(Wh), "e4m3": ops.E4m3WeightMap.quantize(Wh)}
    x = torch.randn((M, 4096), generator=g, device=dev).half()
    act = torch.empty((M, 11008), dtype=torch.float16, device=dev)

    def fwd(layers, head):
        h = x
        for qkv, o, gu, d in layers:
            ops.stream_linear(h, qkv, workspace=ws)
            h = ops.stream_linear(x, o, workspace=ws)
            ops.stream_linear(h, gu, silu=True, out=act, workspace=ws)
            h = ops.stream_linear(act, d, workspace=ws)
        return ops.stream_linear(h, head, out_fp32=True, workspace=ws)

    graphs = {}
    for kind, layers in (("fp16", layers16), ("e4m3", layers8)):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fwd(layers, heads[kind])
        torch.cuda.current_stream().wait_stream(s)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fwd(layers, heads[kind])
        graphs[kind] = gr
    t = alternate({k: gr.replay for k, gr in graphs.items()}, max(args.iters // 10, 10), args.rounds)
    b16 = (L * sum(SHAPES[n][0] * SHAPES[n][1] for n in ("qkv", "o", "gate_up", "down")) + 32000 * 4096) * 2
    b8 = L * sum(SHAPES[n][0] * (SHAPES[n][1] + 1) for n in ("qkv", "o", "gate_up", "down")) + 32000 * 4097
    ms16, ms8 = median(t["fp16"]), median(t["e4m3"])
    return {"M": M, "launches": L * 4 + 1, "fp16_ms": round(ms16, 4), "e4m3_ms": round(ms8, 4), "e4m3_over_fp16": round(ms8 / ms16, 3),
            "fp16_TBps": round(b16 / ms16 / 1e9, 3), "e4m3_TBps": round(b8 / ms8 / 1e9, 3),
            "fp16_ms_all": [round(v, 4) for v in t["fp16"]], "e4m3_ms_all": [round(v, 4) for v in t["e4m3"]]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8, help="timed TriForce outer steps of the workload")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ar-steps", dest="ar_steps", type=int, default=24)
    ap.add_argument("--prefill", type=int, default=124928)
    ap.add_argument("--gen-len", dest="gen_len", type=int, default=1024, help="KV capacity reserved for generated tokens")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-workload", dest="no_workload", action="store_true", help="time the projections only")
    ap.add_argument("--weights", choices=["fp16", "e4m3"], default=None, help=argparse.SUPPRESS)  # one subprocess leg
    ap.add_argument("--kv", choices=["fp16", "e4m3"], default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weights_e4m3 needs a CUDA device")
    if args.weights:
        print(json.dumps(workload(args)))
        return
    legs = {}
    if not args.no_workload:  # each leg in a subprocess of its own, while this process holds no device memory
        legs = {"what": f"llama-7B-128K (random-init) + llama-68M draft, prefill {args.prefill}, budget 4096, chunk 8, "
                        f"gamma 6, T 0.6, top_p 0.9; whole-loop device graph; {args.steps} timed outer steps"}
        for w, kv in (("fp16", "fp16"), ("e4m3", "fp16"), ("e4m3", "e4m3")):
            cmd = [sys.executable, os.path.abspath(__file__), "--weights", w, "--kv", kv] + [
                f"--{k}={getattr(args, k.replace('-', '_'))}" for k in ("steps", "warmup", "ar-steps", "prefill", "gen-len", "seed")]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"the {w}-weight / {kv}-KV workload failed (rc {p.returncode}):\n{p.stderr[-4000:]}")
            legs[f"{w}_weights_{kv}_kv"] = json.loads(p.stdout.strip().splitlines()[-1])
    res = {"metric": "stream_linear_e4m3", "card": card(), "launches": launches(args)}
    torch.cuda.empty_cache()
    res["verify_forward_projections"] = forward_graph(args)
    if legs:
        res["workload"] = legs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
