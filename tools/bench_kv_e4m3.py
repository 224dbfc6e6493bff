"""E4M3 full-KV store against fp16, in one command:

1. the verify launch: tf_verify_attn_e4m3 against the fp16 launches (tf_verify_attn at 32 MHA heads, tf_verify_attn_gqa at
   32 query / 8 KV heads), 8 rows over 124 944 keys of one layer, alternated in the same run and timed with CUDA events;
2. the cfg2 workload (llama-7B-128K with random-init weights + llama-68M draft, prefill 124 928, budget 4096, chunk 8, gamma 6,
   TriForce through the whole-loop device graph) with kv_dtype fp16 and e4m3: tokens/s, ms per outer step, autoregressive
   ms/token, prefill seconds and peak device memory.  The fp16 store alone peaks near 80 GB, so each dtype runs in a
   subprocess of its own.

Prints one JSON line with the card's name and power limit beside the numbers.

    python tools/bench_kv_e4m3.py [--iters 200] [--rounds 5] [--steps 8] [--no-workload]

Bandwidth is algorithmic bytes over time: kv_len·Hkv·d·2 (K and V) bytes per element width, plus kv_len·Hkv·2 exponent bytes
for e4m3.
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

from oracle import triforce_oracle as orc  # noqa: E402
from triforce_b200 import ops  # noqa: E402


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
    """The cfg2 TriForce workload on a `a.workload` full-KV store (see the module docstring)."""
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
    target = LlamaModel(cfg_t, cuda_state_dict(cfg_t, seed=1, device=dev), device=dev)
    draft = LlamaModel(cfg_d, cuda_state_dict(cfg_d, seed=2, device=dev), device=dev, is_draft=True)
    torch.cuda.empty_cache()
    cache = FlashSimpleCache(target, P + a.gen_len + 16, kv_dtype=a.workload)
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
    return {"kv_dtype": a.workload, "tokens_per_s": tokens / (ms * 1e-3), "ms_per_step": ms / a.steps, "tokens_per_step": tokens / a.steps,
            "steps": a.steps, "ar_ms_per_token": ar_ms, "prefill_seconds": prefill_s,
            "peak_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9}


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
    ap.add_argument("--no-workload", dest="no_workload", action="store_true", help="time the verify launch only")
    ap.add_argument("--workload", choices=["fp16", "e4m3"], default=None, help=argparse.SUPPRESS)  # one subprocess leg
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_e4m3 needs a CUDA device")
    if args.workload:
        print(json.dumps(workload(args)))
        return
    # the workload legs first, each in a subprocess of its own, while this process holds no device memory: the fp16 store
    # alone needs nearly the whole card
    legs = {}
    if not args.no_workload:
        legs = {"what": f"llama-7B-128K (random-init) + llama-68M draft, prefill {args.prefill}, budget 4096, chunk 8, "
                        f"gamma 6, T 0.6, top_p 0.9; whole-loop device graph; {args.steps} timed outer steps"}
        for kind in ("fp16", "e4m3"):
            cmd = [sys.executable, os.path.abspath(__file__), "--workload", kind] + [
                f"--{k}={getattr(args, k.replace('-', '_'))}" for k in ("steps", "warmup", "ar-steps", "prefill", "gen-len", "seed")]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"the {kind} workload failed (rc {p.returncode}):\n{p.stderr[-4000:]}")
            legs[kind] = json.loads(p.stdout.strip().splitlines()[-1])
    dev = "cuda"
    R, kv_len, d = 8, 124944, 128
    cap = (kv_len + 63) // 64 * 64
    scale = orc.softmax_scale_fp16(d)
    g = torch.Generator(device=dev).manual_seed(0)
    cases = {}
    for name, Hq, Hkv in (("mha32", 32, 32), ("gqa32x8", 32, 8)):
        K = torch.randn((1, Hkv, cap, d), generator=g, device=dev).half()
        V = torch.randn((1, Hkv, cap, d), generator=g, device=dev).half()
        st = ops.E4m3Store.empty(1, Hkv, cap, d, dev)
        ops.kv_quantize_e4m3(K[0], st.k_codes[0], st.k_exp[0], 0, cap)
        ops.kv_quantize_e4m3(V[0], st.v_codes[0], st.v_exp[0], 0, cap)
        maps = ops.KVTensorMaps(K, V)
        q = torch.randn((R, Hq, d), generator=g, device=dev).half()
        out = torch.empty_like(q)
        ws16 = ops.verify_attn_workspace(R, Hq, d, dev) if Hq == Hkv else ops.verify_attn_gqa_workspace(Hq, Hkv, d, dev)
        ws8 = ops.verify_attn_gqa_workspace(Hq, Hkv, d, dev)
        if Hq == Hkv:
            fp16 = lambda q=q, maps=maps, out=out, ws=ws16, H=Hq: ops.verify_attn(q, maps, 0, kv_len, R, H, d, scale, out, ws)
        else:
            fp16 = lambda q=q, maps=maps, out=out, ws=ws16, Hq=Hq, Hkv=Hkv: ops.verify_attn_gqa(q, maps, 0, kv_len, R, Hq, Hkv, d, scale,
                                                                                             out, ws)
        e4m3 = lambda q=q, st=st, out=out, ws=ws8, Hq=Hq, Hkv=Hkv: ops.verify_attn_e4m3(q, st, 0, kv_len, R, Hq, Hkv, d, scale, out, ws)
        cases[name] = dict(fp16=fp16, e4m3=e4m3, Hkv=Hkv, keep=(K, V, st, maps))
    res = {"metric": "verify_attn_e4m3_launch", "R": R, "kv_len": kv_len, "d": d, "card": card(), "cases": {}}
    for name, c in cases.items():
        for f in (c["fp16"], c["e4m3"]):
            for _ in range(20):
                f()
        torch.cuda.synchronize()
        times = {"fp16": [], "e4m3": []}
        for _ in range(args.rounds):  # alternate the two launches, one timed window each per round
            for kind in ("fp16", "e4m3"):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    c[kind]()
                b.record()
                b.synchronize()
                times[kind].append(a.elapsed_time(b) / args.iters)
        Hkv = c["Hkv"]
        bytes_ = {"fp16": kv_len * Hkv * d * 2 * 2, "e4m3": kv_len * Hkv * (d + 1) * 2}
        row = {}
        for kind in ("fp16", "e4m3"):
            ms = sorted(times[kind])[len(times[kind]) // 2]
            row[kind] = {"ms": round(ms, 4), "ms_all": [round(t, 4) for t in times[kind]], "TBps": round(bytes_[kind] / ms / 1e9, 3)}
        row["e4m3_over_fp16"] = round(row["e4m3"]["ms"] / row["fp16"]["ms"], 3)
        res["cases"][name] = row
    if legs:
        res["workload"] = legs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
