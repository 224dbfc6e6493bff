"""Greedy decoding (temperature 0) against sampling (temperature 0.6), in one command:

1. the cfg2 workload (llama-7B-128K target + llama-68M draft, random-init weights moved to acceptance-calibrated ones with
   synth.retune_agreement at alpha 0.003 for both, prefill 124 928, budget 4096, chunk 8, gamma 6, TriForce through the
   whole-loop device graph) at T = 0 and at T = 0.6, each leg in a subprocess of its own.  Reports ms per outer step,
   tokens per step and tokens/s;
2. tf_norm_logits on [gamma + 2, 32000] and [1, 32000] fp32 rows at T = 0 and T = 0.6 (top_p 0.9), alternated in the same
   run and timed with CUDA events over many launches.

Prints one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/bench_greedy.py [--steps 16] [--warmup 2] [--iters 500] [--rounds 5] [--no-workload]
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

GAMMA, V = 6, 32000
TEMPS = (0.0, 0.6)


def norm_logits_timing(args) -> dict:
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    out = {}
    for rows in (GAMMA + 2, 1):
        x = torch.randn((rows, V), generator=g, device="cuda") * 3
        o = {t: torch.empty_like(x) for t in TEMPS}
        fns = {f"T{t}": (lambda t=t: ops.norm_logits(x, t, 0.9, out=o[t])) for t in TEMPS}
        t = alternate(fns, args.iters, args.rounds)
        out[f"rows{rows}"] = {k: {"us": round(median(v) * 1e3, 2), "us_all": [round(u * 1e3, 2) for u in v]} for k, v in t.items()}
    return out


def workload(a) -> dict:
    """One cfg2 leg at temperature `a.temp` (see the module docstring)."""
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from triforce_b200.config import named_config
    from triforce_b200.device_loop import DeviceLoopRun
    from triforce_b200.engine import GraphInferenceEngine
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import cuda_state_dict, retune_agreement

    dev = torch.device("cuda", 0)
    torch.manual_seed(a.seed)
    P, B, chunk, top_p = a.prefill, 4096, 8, 0.9
    cfg_t, cfg_d = named_config("llama-7B-128K"), named_config("llama-68M")
    target = LlamaModel(cfg_t, cuda_state_dict(cfg_t, seed=1, device=dev), device=dev)
    draft = LlamaModel(cfg_d, cuda_state_dict(cfg_d, seed=2, device=dev), device=dev, is_draft=True)
    retune_agreement(target, draft, a.alpha, a.alpha, {})
    torch.cuda.empty_cache()
    cache = FlashSimpleCache(target, P + a.gen_len + 16)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=GAMMA, chunk_size=chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - GAMMA, gamma=GAMMA)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(GAMMA, probs=True, temperature=a.temp, top_p=top_p)
    g = torch.Generator().manual_seed(a.seed)
    input_ids = torch.randint(0, cfg_t.vocab_size, (1, P), generator=g).to(dev)
    tok = type("Tok", (), {"eos_token_id": 2, "decode": lambda self, *x, **k: ""})()
    with torch.inference_mode():
        run = DeviceLoopRun(tok, ge, gamma=GAMMA, top_p=top_p, temperature=a.temp, seed=a.seed, max_new=a.gen_len)
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
    return {"temperature": a.temp, "tokens_per_s": tokens / (ms * 1e-3), "ms_per_step": ms / a.steps,
            "tokens_per_step": tokens / a.steps, "steps": a.steps, "acceptance_rate": run.acceptance_rate,
            "prefill_seconds": prefill_s}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=16, help="timed TriForce outer steps per leg")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--prefill", type=int, default=124928)
    ap.add_argument("--gen-len", dest="gen_len", type=int, default=1024, help="KV capacity reserved for generated tokens")
    ap.add_argument("--alpha", type=float, default=0.003, help="agreement alpha of target and draft (synth.retune_agreement)")
    ap.add_argument("--iters", type=int, default=500, help="tf_norm_logits launches per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-workload", dest="no_workload", action="store_true", help="time tf_norm_logits only")
    ap.add_argument("--temp", type=float, default=None, help=argparse.SUPPRESS)  # one subprocess leg
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_greedy needs a CUDA device")
    if args.temp is not None:
        print(json.dumps(workload(args)))
        return
    legs = {}
    if not args.no_workload:  # each leg in a subprocess of its own, while this process holds no device memory
        legs = {"what": f"llama-7B-128K + llama-68M draft, retune_agreement alpha {args.alpha}, prefill {args.prefill}, budget 4096, "
                        f"chunk 8, gamma 6, top_p 0.9; whole-loop device graph; {args.steps} timed outer steps"}
        for t in TEMPS:
            cmd = [sys.executable, os.path.abspath(__file__), "--temp", str(t)] + [
                f"--{k}={getattr(args, k.replace('-', '_'))}" for k in ("steps", "warmup", "prefill", "gen-len", "alpha", "seed")]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"the T = {t} leg failed (rc {p.returncode}):\n{p.stderr[-4000:]}")
            legs[f"T{t}"] = json.loads(p.stdout.strip().splitlines()[-1])
    res = {"metric": "greedy_decoding", "card": card(), "norm_logits": norm_logits_timing(args)}
    if legs:
        res["workload"] = legs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
