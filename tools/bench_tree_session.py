"""Follow-up turns on the Sequoia tree path against a fresh prefill, at cfg5 shapes, in one command.

Each leg runs in a subprocess of its own: llama-13B-128K target (40 layers, seeded random-init weights), SingleGpuLlama, budget
8192, chunk 8, the 512-node tree, T 0.6, top_p 0.9, through triforce_b200.session.TreeSession (Philox noise, fp32 race redrawn
every round).
  * e4m3: E4M3 weights and full-KV store, prompt 129 024.  The 128K model has 131 072 RoPE positions; 130 048 prompt tokens
    would leave 1 024 for the turns and the 1 024-token follow-up would not fit;
  * fp16: fp16 weights and full-KV store, prompt 49 152.
A leg times the fresh prefill and first token, turn 1, then follow-ups of 64, 256 and 1024 tokens.  A follow-up's time to first
token runs from the start of append to the first sampled token, split into extend, re-selection and first sample.  ms per
round is the host time of each tree round (growth + verify + compaction), median over the rounds of the turn after the first.
Random-init weights accept almost nothing, so tokens per round is printed beside the times.

Prints one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/bench_tree_session.py [--gen 8]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_session import _Clock  # noqa: E402
from bench_weights_e4m3 import card  # noqa: E402

BUDGET, CHUNK, TEMP, TOP_P = 8192, 8, 0.6, 0.9
FOLLOW_UPS = (64, 256, 1024)
LEGS = {"e4m3": 129024, "fp16": 49152}


def leg(a) -> dict:
    from triforce_b200 import session as session_mod
    from triforce_b200.config import named_config
    from triforce_b200.session import TreeSession
    from triforce_b200.spectree import load_grow_map
    from triforce_b200.synth import cuda_state_dict
    from triforce_b200.tp import SingleGpuLlama

    fmt, P = a.leg, LEGS[a.leg]
    dev = torch.device("cuda", 0)
    cfg = named_config("llama-13B-128K")
    gm = load_grow_map("512")
    turns = 1 + len(FOLLOW_UPS)
    max_context = P + sum(FOLLOW_UPS) + turns * (a.gen + 32)
    llm = SingleGpuLlama("llama-13B-128K", local_rank=0, world_size=1, prefill=P, gen_len=64, retrieval_budget=BUDGET,
                         retrieval_chunk_size=CHUNK, temperature=TEMP, top_p=TOP_P, config=cfg, tree_size=gm["size"],
                         kv_dtype=fmt, weight_dtype=fmt, max_context=max_context)
    llm.init_parameters(state_dict=cuda_state_dict(cfg, seed=1, device=dev, host=True), cuda_graphs=False)
    torch.cuda.empty_cache()
    g = torch.Generator().manual_seed(a.seed)
    ids = torch.randint(3, cfg.vocab_size, (P + sum(FOLLOW_UPS),), generator=g)
    s = TreeSession(llm, grow_map=gm)
    clock = _Clock()
    for name, tag in (("_extend", "extend"), ("_reselect", "reselect"), ("_first_token", "first_token")):
        clock.wrap(s, name, tag)
    clock.wrap(session_mod, "tree_round", "round")

    def turn(seed):
        toks = s.generate(a.gen, temperature=TEMP, top_p=TOP_P, seed=seed)
        log = clock.take()
        rounds = [x for tag, x, _ in log if tag == "round"][1:]
        t = s.last_turn
        return log, {"ms_per_round": 1e3 * statistics.median(rounds) if rounds else None, "timed_rounds": len(rounds),
                     "tokens": len(toks), "tokens_per_round": t.tokens_per_round, "stop": t.stop}

    out = {"format": fmt, "prefill": P}
    with torch.inference_mode():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.prefill(ids[:P])
        torch.cuda.synchronize()
        prefill_s = time.perf_counter() - t0
        log, t1 = turn(1)
        first = next(x for tag, x, _ in log if tag == "first_token")
        out["fresh"] = {"prefill_s": prefill_s, "first_token_s": prefill_s + first}
        out["turn1"] = t1
        off = P
        for n in FOLLOW_UPS:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s.append(ids[off:off + n])
            off += n
            log, t2 = turn(100 + n)
            end_first = next(e for tag, _, e in log if tag == "first_token")
            parts = {tag: 1e3 * sum(x for t, x, _ in log if t == tag) for tag in ("extend", "reselect", "first_token")}
            out[f"follow_up_{n}"] = {**{f"{k}_ms": v for k, v in parts.items()}, "time_to_first_token_ms": 1e3 * (end_first - t0),
                                     "turn": t2, "boundary": llm.retrieval_cache.prefill, "length": s.length}
        out["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gen", type=int, default=8, help="tokens generated per turn")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--leg", choices=tuple(LEGS), default=None, help=argparse.SUPPRESS)  # one subprocess leg
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tree_session needs a CUDA device")
    if args.leg is not None:
        print(json.dumps(leg(args)))
        return
    res = {"metric": "tree_follow_up_turns", "card": card(),
           "what": f"llama-13B-128K (random-init), SingleGpuLlama, budget {BUDGET}, chunk {CHUNK}, 512-node tree, T {TEMP}, "
                   f"top_p {TOP_P}, TreeSession, {args.gen} tokens per turn"}
    for fmt in LEGS:  # each leg in a subprocess of its own, while this process holds no device memory
        cmd = [sys.executable, os.path.abspath(__file__), "--leg", fmt, f"--gen={args.gen}", f"--seed={args.seed}"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            res[fmt] = {"error": f"rc {p.returncode}", "stderr": p.stderr[-3000:]}
            continue
        r = json.loads(p.stdout.strip().splitlines()[-1])
        fresh = r["fresh"]["first_token_s"] * 1e3
        for n in FOLLOW_UPS:
            r[f"follow_up_{n}"]["first_token_speedup"] = fresh / r[f"follow_up_{n}"]["time_to_first_token_ms"]
        res[fmt] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
