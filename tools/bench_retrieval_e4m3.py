"""E4M3 retrieval cache against fp16, in one command:

1. the retrieval-verify attention of one layer at the 7B shapes (32 heads, d = 128), budgets 4096, 8192 and 12288, R = 7 and 17
   rows (gamma 6 and 16): tf_verify_attn with clean_keys = budget on the fp16 cache against tf_verify_attn_e4m3_clean on the E4M3
   cache, alternated in the same run and timed with CUDA events over many launches (back to back, so each launch is
   programmatically chained to the previous one as in a forward);
2. the whole retrieval-verify forward of the 7B target (32 layers, random-init fp16 weights) captured as one CUDA graph, fp16
   cache against E4M3 cache, alternated, at the same budgets and rows;
3. the cfg2 workload (llama-7B-128K + llama-68M draft with acceptance-calibrated weights, synth.agreement_state_dicts at
   alpha 0.003 for both, prefill 124 928, chunk 8, gamma 6, TriForce through the whole-loop device graph), each leg in a
   subprocess of its own: fp16 everything; E4M3 retrieval cache only; E4M3 retrieval cache, store and weights; E4M3
   retrieval cache at budget 8192.  Reports ms per outer step, tokens per step, tokens/s, peak memory and prefill seconds.

Prints one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/bench_retrieval_e4m3.py [--iters 200] [--rounds 5] [--steps 8] [--no-workload]

Bandwidth is algorithmic K and V bytes over time: slots * 32 heads * 128 * 2 (K and V) * 2 B for fp16, and * (128 + 1) B for E4M3
(codes and the exponent byte of each row), per layer.
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

from bench_weights_e4m3 import alternate, card, median  # noqa: E402
from triforce_b200 import ops  # noqa: E402

H, D = 32, 128
BUDGETS = (4096, 8192, 12288)
ROWS = (7, 17)


def kv_bytes(slots: int, dtype: str, layers: int = 1) -> int:
    return layers * 2 * H * slots * (D * 2 if dtype == "fp16" else D + 1)


def _random_e4m3(store: ops.E4m3Store, g) -> None:
    """Finite random codes (0x7F / 0xFF are NaN) and exponents of typical K / V rows."""
    for c in (store.k_codes, store.v_codes):
        c.copy_(torch.randint(0, 0x7F, c.shape, generator=g, device=c.device, dtype=torch.uint8)
                | (torch.randint(0, 2, c.shape, generator=g, device=c.device, dtype=torch.uint8) << 7))
    for e in (store.k_exp, store.v_exp):
        e.copy_(torch.randint(-8, -3, e.shape, generator=g, device=e.device, dtype=torch.int8))


def attention(args) -> dict:
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(args.seed)
    scale = D ** -0.5
    out = {}
    for budget in BUDGETS:
        for R in ROWS:
            slots = budget + R
            cap = -(-slots // ops.VERIFY_BOX_KEYS) * ops.VERIFY_BOX_KEYS
            K = (torch.randn((1, H, slots, D), generator=g, device=dev) * 0.5).half()
            V = torch.randn((1, H, slots, D), generator=g, device=dev).half()
            maps = ops.KVTensorMaps(K, V)
            st = ops.E4m3Store.empty(1, H, cap, D, dev)
            _random_e4m3(st, g)
            q = torch.randn((R, H, D), generator=g, device=dev).half()
            o16, o8 = torch.empty_like(q), torch.empty_like(q)
            ws16 = ops.verify_attn_workspace(ops.VERIFY_MAX_ROWS, H, D, dev)
            ws8 = ops.verify_attn_workspace(ops.VERIFY_MAX_ROWS, H, D, dev)
            f16 = lambda: ops.verify_attn(q, maps, 0, slots, R, H, D, scale, o16, ws16, clean_keys=budget)
            f8 = lambda: ops.verify_attn_e4m3(q, st, 0, slots, R, H, H, D, scale, o8, ws8, clean_keys=budget)
            t = alternate({"fp16": f16, "e4m3": f8}, args.iters, args.rounds)
            ms16, ms8 = median(t["fp16"]), median(t["e4m3"])
            out[f"B{budget}_R{R}"] = {"slots": slots, "fp16_us": round(ms16 * 1e3, 2), "e4m3_us": round(ms8 * 1e3, 2),
                                      "e4m3_over_fp16": round(ms8 / ms16, 3),
                                      "fp16_TBps": round(kv_bytes(slots, "fp16") / ms16 / 1e9, 3),
                                      "e4m3_TBps": round(kv_bytes(slots, "e4m3") / ms8 / 1e9, 3),
                                      "fp16_us_all": [round(v * 1e3, 2) for v in t["fp16"]],
                                      "e4m3_us_all": [round(v * 1e3, 2) for v in t["e4m3"]]}
            del K, V, maps, st
            torch.cuda.empty_cache()
    return out


def forward(args) -> dict:
    """The retrieval-verify forward of the 32-layer 7B target as one CUDA graph (forward_target with spec=True)."""
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache
    from triforce_b200.config import named_config
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import cuda_state_dict

    dev = torch.device("cuda", 0)
    cfg = named_config("llama-7B-128K")
    target = LlamaModel(cfg, cuda_state_dict(cfg, seed=1, device=dev), device=dev)
    full = FlashSimpleCache(target, 64)  # the retrieval verify reads no full-KV row
    g = torch.Generator(device=dev).manual_seed(args.seed + 1)
    out = {}
    for budget in BUDGETS:
        for R in ROWS:
            graphs = {}
            for kind in ("fp16", "e4m3"):
                gc = RetrievalCache(target, max_budget=budget, prefill=budget, gamma=R - 1, chunk_size=8, kv_dtype=kind)
                if kind == "fp16":
                    gc.key_store.normal_(0, 0.5, generator=g)
                    gc.value_store.normal_(0, 1.0, generator=g)
                else:
                    _random_e4m3(gc.e4m3, g)
                ids = torch.randint(0, cfg.vocab_size, (1, R), generator=g, device=dev)
                pos = torch.arange(budget, budget + R, device=dev).unsqueeze(0)
                fn = lambda gc=gc, ids=ids, pos=pos: target.forward_target(ids, full, gc, pos, spec=True)
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s), torch.inference_mode():
                    for _ in range(2):
                        fn()
                torch.cuda.current_stream().wait_stream(s)
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr), torch.inference_mode():
                    fn()
                graphs[kind] = (gr, gc)
            t = alternate({k: v[0].replay for k, v in graphs.items()}, max(args.iters // 20, 5), args.rounds)
            ms16, ms8 = median(t["fp16"]), median(t["e4m3"])
            out[f"B{budget}_R{R}"] = {"fp16_ms": round(ms16, 4), "e4m3_ms": round(ms8, 4), "e4m3_over_fp16": round(ms8 / ms16, 3),
                                      "kv_bytes_fp16": kv_bytes(budget + R, "fp16", cfg.num_hidden_layers),
                                      "kv_bytes_e4m3": kv_bytes(budget + R, "e4m3", cfg.num_hidden_layers),
                                      "fp16_ms_all": [round(v, 4) for v in t["fp16"]], "e4m3_ms_all": [round(v, 4) for v in t["e4m3"]]}
            del graphs
            torch.cuda.empty_cache()
    return out


def workload(a) -> dict:
    """One cfg2 leg: `a.retrieval` cache, `a.kv` store, `a.weights` weights, budget `a.budget` (see the module docstring)."""
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from triforce_b200.config import named_config
    from triforce_b200.device_loop import DeviceLoopRun
    from triforce_b200.engine import GraphInferenceEngine
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import agreement_state_dicts

    dev = torch.device("cuda", 0)
    torch.manual_seed(a.seed)
    P, B, chunk, gamma, temp, top_p = a.prefill, a.budget, 8, 6, 0.6, 0.9
    cfg_t, cfg_d = named_config("llama-7B-128K"), named_config("llama-68M")
    tsd, dsd = agreement_state_dicts(cfg_t, cfg_d, a.alpha, a.alpha, seed=0, device=dev)
    target = LlamaModel(cfg_t, tsd, device=dev, weight_dtype=a.weights)
    draft = LlamaModel(cfg_d, dsd, device=dev, is_draft=True)
    del tsd, dsd
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    cache = FlashSimpleCache(target, P + a.gen_len + 16, kv_dtype=a.kv)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=gamma, chunk_size=chunk, kv_dtype=a.retrieval)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(gamma, probs=True, temperature=temp, top_p=top_p)
    g = torch.Generator().manual_seed(a.seed)
    input_ids = torch.randint(0, cfg_t.vocab_size, (1, P), generator=g).to(dev)
    tok = type("Tok", (), {"eos_token_id": 2, "decode": lambda self, *x, **k: ""})()
    with torch.inference_mode():
        run = DeviceLoopRun(tok, ge, gamma=gamma, top_p=top_p, temperature=temp, seed=a.seed, max_new=a.gen_len)
        torch.cuda.synchronize()
        t0 = time.time()
        run.prefill(input_ids)
        torch.cuda.synchronize()
        prefill_s = time.time() - t0
        for _ in range(a.warmup):
            run.step()
        torch.cuda.synchronize()
        n0 = run.n
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            run.step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        tokens = run.n - n0
    return {"retrieval_dtype": a.retrieval, "kv_dtype": a.kv, "weight_dtype": a.weights, "budget": B,
            "tokens_per_s": tokens / (ms * 1e-3), "ms_per_step": ms / a.steps, "tokens_per_step": tokens / a.steps, "steps": a.steps,
            "acceptance_rate": run.acceptance_rate, "prefill_seconds": prefill_s,
            "peak_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9}


LEGS = (("fp16", "fp16", "fp16", 4096), ("e4m3", "fp16", "fp16", 4096), ("e4m3", "e4m3", "e4m3", 4096), ("e4m3", "fp16", "fp16", 8192))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8, help="timed TriForce outer steps of the workload")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--prefill", type=int, default=124928)
    ap.add_argument("--gen-len", dest="gen_len", type=int, default=1024, help="KV capacity reserved for generated tokens")
    ap.add_argument("--alpha", type=float, default=0.003, help="agreement alpha of target and draft (synth.agreement_state_dicts)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-workload", dest="no_workload", action="store_true", help="time the attention and the forward only")
    ap.add_argument("--retrieval", choices=["fp16", "e4m3"], default=None, help=argparse.SUPPRESS)  # one subprocess leg
    ap.add_argument("--kv", choices=["fp16", "e4m3"], default="fp16", help=argparse.SUPPRESS)
    ap.add_argument("--weights", choices=["fp16", "e4m3"], default="fp16", help=argparse.SUPPRESS)
    ap.add_argument("--budget", type=int, default=4096, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval_e4m3 needs a CUDA device")
    if args.retrieval:
        print(json.dumps(workload(args)))
        return
    legs = {}
    if not args.no_workload:  # each leg in a subprocess of its own, while this process holds no device memory
        legs = {"what": f"llama-7B-128K + llama-68M draft, agreement weights alpha {args.alpha}, prefill {args.prefill}, chunk 8, "
                        f"gamma 6, T 0.6, top_p 0.9; whole-loop device graph; {args.steps} timed outer steps"}
        for r, kv, w, b in LEGS:
            cmd = [sys.executable, os.path.abspath(__file__), "--retrieval", r, "--kv", kv, "--weights", w, "--budget", str(b)] + [
                f"--{k}={getattr(args, k.replace('-', '_'))}" for k in ("steps", "warmup", "prefill", "gen-len", "alpha", "seed")]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"the {r} retrieval / {kv} store / {w} weights / budget {b} leg failed (rc {p.returncode}):\n"
                                 f"{p.stderr[-4000:]}")
            legs[f"retrieval_{r}_kv_{kv}_weights_{w}_budget_{b}"] = json.loads(p.stdout.strip().splitlines()[-1])
    res = {"metric": "retrieval_cache_e4m3", "card": card(), "attention": attention(args)}
    torch.cuda.empty_cache()
    res["retrieval_verify_forward"] = forward(args)
    if legs:
        res["workload"] = legs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
