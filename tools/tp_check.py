#!/usr/bin/env python
"""Tensor-parallel parity check: TriForce_Dist on the tiny golden config, head-sharded over WORLD_SIZE GPUs, replaying a
CounterNoise stream; rank 0 writes the event trace.  Run once with 1 process and once under torchrun with N, then diff:
    python tools/tp_check.py --out gpurun_out/tp1.json
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 tools/tp_check.py --out gpurun_out/tp2.json
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
from triforce_b200.cache import StreamingLLMEvictionCache  # noqa: E402
from triforce_b200.config import named_config  # noqa: E402
from triforce_b200.decoding import TriForce_Dist  # noqa: E402
from triforce_b200.llama import LlamaModel  # noqa: E402
from triforce_b200.rng import CounterNoise  # noqa: E402
from triforce_b200.synth import numpy_prompt, numpy_state_dict  # noqa: E402
from triforce_b200.tp import DistributedLlama  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--gen", type=int, default=0, help="tokens to generate (0 = the golden case's gen_len)")
    ap.add_argument("--case", default="tiny", help="golden case under tests/golden/e2e_<case>.json (same weights, prompt, noise)")
    ap.add_argument("--draft_chunk", type=int, default=64, help="draft prefill chunk: 64 = on-chip (the golden traces), 128 = TP_llama.py:118-126")
    ap.add_argument("--device_loop", type=int, default=0, metavar="SEED",
                    help="instead of replaying the golden trace: run the whole-loop graph (DeviceLoopRun, what bench.py times at every N) and the "
                         "step-wise loop on the same device Philox stream, each on a freshly built sharded engine, and compare their tokens")
    ap.add_argument("--retrieval_dtype", default="fp16", choices=["fp16", "e4m3"], help="the rank-local retrieval cache's format")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    case = json.load(open(os.path.join(REPO, "tests", "golden", f"e2e_{args.case}.json")))["case"]
    args.gen = args.gen or case["gen_len"]
    ts, ds = named_config(case["target"]), named_config(case["draft"])
    gamma, P, B = case["gamma"], case["prefill"], case["budget"]

    def build():
        draft = LlamaModel(ds, numpy_state_dict(ds, case["draft_seed"]), device=dev, is_draft=True)
        dcache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
        m = DistributedLlama(case["target"], local_rank=rank, world_size=world, prefill=P, gen_len=args.gen + 16, retrieval_budget=B,
                             retrieval_chunk_size=case["chunk"], gamma=gamma, temperature=case["temperature"], top_p=case["top_p"],
                             draft=draft, draft_cache=dcache, config=ts, retrieval_dtype=args.retrieval_dtype)
        m.init_parameters(state_dict=numpy_state_dict(ts, case["target_seed"]))
        m.graph_engine.engine.draft_prefill_chunk = args.draft_chunk
        return m

    ids = numpy_prompt(P, seed=case["prompt_seed"]).to(dev)
    tok = type("T", (), {"eos_token_id": 2, "decode": lambda self, *a, **k: ""})()
    if args.device_loop:
        from triforce_b200.decoding import TriForceRun
        from triforce_b200.device_loop import DeviceLoopRun, PhiloxNoise
        gen = min(args.gen, 32)
        runs = {}
        for kind in ("host", "device"):  # a fresh engine each: both loops must see a FIRST prompt (draft-cache reset quirk)
            ge = build().graph_engine
            if kind == "host":
                r = TriForceRun(tok, ge, gamma=gamma, top_p=case["top_p"], temperature=case["temperature"],
                                noise=PhiloxNoise(dev, args.device_loop), pad_full_verify=True)
            else:
                r = DeviceLoopRun(tok, ge, gamma=gamma, top_p=case["top_p"], temperature=case["temperature"], seed=args.device_loop)
            r.prefill(ids)
            steps = []
            while r.n < gen:
                before = len(r.generated)
                r.step()
                steps.append(list(r.generated[before:]))
            runs[kind] = dict(tokens=[int(t) for t in r.generated], steps=steps, inner=int(r.inner_iterations), accepted=int(r.accepted_count),
                              drafted=int(r.draft_count), seq_len=int(ge.engine.kv_cache.seq_len))
            del r, ge
        if rank == 0:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            json.dump(dict(world=world, mode="device_loop", seed=args.device_loop, identical=runs["host"] == runs["device"], **runs), open(args.out, "w"))
            print(f"[tp_check] world={world} device loop vs step-wise loop: identical={runs['host'] == runs['device']} tokens={len(runs['device']['tokens'])}")
        if world > 1:
            dist.barrier()
            sys.stdout.flush()
            os._exit(0)
        return
    llm = build()
    out = {}
    for call in range(2):
        trace, stats = [], {}
        avg, lat = TriForce_Dist(tok, llm, ids, gamma=gamma, max_len=args.gen, top_p=case["top_p"], temperature=case["temperature"],
                                 noise=CounterNoise(case["noise_seed"]),
                                 trace=trace, stats=stats)
        out[f"call{call}"] = dict(trace=[[a, b] for a, b in trace], avg_tokens=avg, latency=lat, n=stats["n"])
    if rank == 0:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(world=world, **out), open(args.out, "w"))
        print(f"[tp_check] world={world} call0: n={out['call0']['n']} events={len(out['call0']['trace'])} avg_tokens={out['call0']['avg_tokens']:.3f}")
    if world > 1:
        dist.barrier()
        sys.stdout.flush()
        os._exit(0)  # NCCL + captured graphs can stall interpreter teardown


if __name__ == "__main__":
    main()
