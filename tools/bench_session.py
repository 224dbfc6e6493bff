"""Follow-up turns against a fresh prefill, at cfg2 shapes, in one command.

Each leg runs in a subprocess of its own: llama-7B-128K target + llama-68M draft, context 124 928, budget 4096, chunk 8, gamma 6,
top_p 0.9, T 0.6, TriForce through the whole-loop device graph (triforce_b200.session.Session).
  * fp16: fp16 weights, full-KV store and retrieval cache; target and draft moved to acceptance-calibrated weights
    (synth.retune_agreement, alpha 0.003);
  * e4m3: E4M3 weights, full-KV store and retrieval cache; random-init weights (retune_agreement rescales fp16 weights only).
A leg times the fresh prefill, turn 1, then follow-ups of 64, 256 and 1024 tokens.  A follow-up is split into extend, re-selection,
draft feed and the re-capture of the whole-loop graph; its time to first token runs from the start of append to the first
sampled token.  ms per outer step is the host time of each graph launch and read-back after --warmup steps of the turn.
After each follow-up's turn, `Session.score` of the follow-up's ids is timed twice (`score_first_ms`, `score_ms`): it forwards
the pending token and those ids, the rows the append's extend forwarded, and rolls the store back, so the next follow-up starts
from the same state.  The append's own fields are timed before any score, as without scoring.

Prints one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/bench_session.py [--gen 64] [--warmup 2]
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

from bench_weights_e4m3 import card  # noqa: E402

P, BUDGET, CHUNK, GAMMA, TOP_P, TEMP = 124928, 4096, 8, 6, 0.9, 0.6
FOLLOW_UPS = (64, 256, 1024)


class _Clock:
    """Host seconds of wrapped calls, each ended by a device synchronise."""

    def __init__(self):
        self.log = []

    def wrap(self, owner, name, tag):
        orig = getattr(owner, name)

        def timed(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = orig(*a, **k)
            torch.cuda.synchronize()
            self.log.append((tag, time.perf_counter() - t0, time.perf_counter()))
            return out
        setattr(owner, name, timed)

    def take(self):
        out, self.log = self.log, []
        return out


def leg(a) -> dict:
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from triforce_b200.config import named_config
    from triforce_b200.device_loop import DeviceLoop, DeviceLoopRun
    from triforce_b200.engine import GraphInferenceEngine
    from triforce_b200.llama import LlamaModel
    from triforce_b200.session import Session
    from triforce_b200.synth import cuda_state_dict, retune_agreement

    dev = torch.device("cuda", 0)
    fmt = a.leg
    cfg_t, cfg_d = named_config("llama-7B-128K"), named_config("llama-68M")
    target = LlamaModel(cfg_t, cuda_state_dict(cfg_t, seed=1, device=dev, host=fmt == "e4m3"), device=dev, weight_dtype=fmt)
    draft = LlamaModel(cfg_d, cuda_state_dict(cfg_d, seed=2, device=dev), device=dev, is_draft=True)
    if fmt == "fp16":
        retune_agreement(target, draft, 0.003, 0.003, {})
    torch.cuda.empty_cache()
    # room for the scores after each follow-up too: the pending token and the largest follow-up's ids
    slots = P + sum(FOLLOW_UPS) + max(FOLLOW_UPS) + 1 + 8 * (a.gen + 2 * GAMMA)
    cache = FlashSimpleCache(target, slots, kv_dtype=fmt)
    graph_cache = RetrievalCache(target, max_budget=BUDGET, prefill=P, gamma=GAMMA, chunk_size=CHUNK, kv_dtype=fmt,
                                 max_context=slots // CHUNK * CHUNK)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - GAMMA, gamma=GAMMA)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(GAMMA, probs=True, temperature=TEMP, top_p=TOP_P)
    g = torch.Generator().manual_seed(a.seed)
    ids = torch.randint(3, cfg_t.vocab_size, (P + sum(FOLLOW_UPS),), generator=g)
    tok = type("Tok", (), {"eos_token_id": 2, "decode": lambda self, *x, **k: ""})()
    s = Session(ge, gamma=GAMMA, tokenizer=tok)
    clock = _Clock()
    for name, tag in (("_extend", "extend"), ("_reselect", "reselect"), ("_feed_draft", "draft_feed")):
        clock.wrap(s, name, tag)
    clock.wrap(DeviceLoop, "__init__", "capture")
    clock.wrap(DeviceLoopRun, "start", "first_token")
    clock.wrap(DeviceLoopRun, "step", "step")

    def turn(seed):
        toks = s.generate(a.gen, temperature=TEMP, top_p=TOP_P, seed=seed, device_loop=True)
        log = clock.take()
        steps = [x for tag, x, _ in log if tag == "step"][a.warmup:]
        r = s.last_run
        return log, {"ms_per_step": 1e3 * sum(steps) / max(len(steps), 1), "timed_steps": len(steps), "tokens": len(toks),
                     "tokens_per_step": (len(toks) - 1) / max(r.steps, 1), "acceptance_rate": r.acceptance_rate}

    out = {"format": fmt}
    with torch.inference_mode():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.prefill(ids[:P])
        torch.cuda.synchronize()
        prefill_s = time.perf_counter() - t0
        log, t1 = turn(1)
        cap = sum(x for tag, x, _ in log if tag == "capture")
        first = next(x for tag, x, _ in log if tag == "first_token")
        out["fresh"] = {"prefill_s": prefill_s, "capture_ms": 1e3 * cap, "first_token_s": prefill_s + cap + first}
        out["turn1"] = t1
        off = P
        for n in FOLLOW_UPS:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s.append(ids[off:off + n])
            off += n
            log, t2 = turn(100 + n)
            score_ms = []
            for _ in range(2):
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                s.score(ids[off - n:off])
                torch.cuda.synchronize()
                score_ms.append(1e3 * (time.perf_counter() - t1))
            end_first = next(e for tag, _, e in log if tag == "first_token")
            parts = {tag: 1e3 * sum(x for t, x, _ in log if t == tag) for tag in ("extend", "reselect", "draft_feed", "capture")}
            out[f"follow_up_{n}"] = {**{f"{k}_ms": v for k, v in parts.items()}, "first_token_ms": 1e3 * (end_first - t0),
                                     "score_first_ms": score_ms[0], "score_ms": score_ms[1],
                                     "turn": t2, "boundary": graph_cache.prefill, "length": s.length}
        out["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gen", type=int, default=64, help="tokens generated per turn")
    ap.add_argument("--warmup", type=int, default=2, help="outer steps of each turn left out of ms per step")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--leg", choices=("fp16", "e4m3"), default=None, help=argparse.SUPPRESS)  # one subprocess leg
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_session needs a CUDA device")
    if args.leg is not None:
        print(json.dumps(leg(args)))
        return
    res = {"metric": "follow_up_turns", "card": card(),
           "what": f"llama-7B-128K + llama-68M, context {P}, budget {BUDGET}, chunk {CHUNK}, gamma {GAMMA}, T {TEMP}, top_p {TOP_P}, "
                   f"whole-loop device graph, {args.gen} tokens per turn"}
    for fmt in ("fp16", "e4m3"):  # each leg in a subprocess of its own, while this process holds no device memory
        cmd = [sys.executable, os.path.abspath(__file__), "--leg", fmt, f"--gen={args.gen}", f"--warmup={args.warmup}",
               f"--seed={args.seed}"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            res[fmt] = {"error": f"rc {p.returncode}", "stderr": p.stderr[-3000:]}
            continue
        r = json.loads(p.stdout.strip().splitlines()[-1])
        fresh = r["fresh"]["first_token_s"] * 1e3
        for n in FOLLOW_UPS:
            r[f"follow_up_{n}"]["first_token_speedup"] = fresh / r[f"follow_up_{n}"]["first_token_ms"]
        res[fmt] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
