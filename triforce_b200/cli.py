"""Command-line front ends behind the reference's three entry points (`test/on_chip.py`, `test/offloading_TP.py`,
`test/offloading_seqouia.py`): the same flags with the same defaults, the same measurement flow and report lines, on the
GPU-native engine.  The scripts under `test/` are one-line wrappers around the `run_*` functions here.

Offline by design (no HF hub, no tokenizer, no dataset files on the box): models are random-init with the named shapes
unless `--target_path` / `--draft_path` point at local HF checkpoints, and the prompt is synthetic token ids.
`--on_chip` of the TP scripts is accepted and ignored — the engine keeps the whole KV in HBM.
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from typing import List, Optional

import numpy as np
import torch

# (flag, kwargs) in the order of the reference's argparse blocks: on_chip.py:21-40, offloading_TP.py:26-44,
# offloading_seqouia.py:41-58.  Defaults are the reference's.
_COMMON_TP_FLAGS = [
    ("--target", dict(type=str, default="lwm-128K", help="target model")),
    ("--verbose", dict(action="store_true", help="verbose")),
    ("--prefill", dict(type=int, default=130048, help="prefill length")),
    ("--gen_len", dict(type=int, default=256, help="generation length")),
    ("--temp", dict(type=float, default=0.6, help="temperature")),
    ("--top_p", dict(type=float, default=0.9, help="top p")),
    ("--dataset", dict(type=str, default="demo", help="dataset")),
    ("--on_chip", dict(type=int, default=0, help="on chip layers (ignored: everything is on chip)")),
    ("--budget", dict(type=int, default=12288)),
    ("--baseline", dict(action="store_true", help="baseline")),
    ("--file", dict(type=str, default="")),
    ("--seed", dict(type=int, default=1, help="seed")),
]
FLAGS = {
    "on_chip": [
        ("--target", dict(type=str, default="llama-7B-128K", help="target model")),
        ("--draft", dict(type=str, default="llama-68M", help="draft model")),
        ("--verbose", dict(action="store_true", help="verbose")),
        ("--prefill", dict(type=int, default=32768, help="prefill length")),
        ("--gen_len", dict(type=int, default=256, help="generation length")),
        ("--gamma", dict(type=int, default=6, help="gamma")),
        ("--dataset", dict(type=str, default="gs", help="dataset")),
        ("--temp", dict(type=float, default=0.6, help="temperature")),
        ("--top_p", dict(type=float, default=0.9, help="top p")),
        ("--budget", dict(type=int, default=4096)),
        ("--draft_cache_budget", dict(type=int, default=256, help="draft cache budget")),
        ("--chunk_size", dict(type=int, default=8, help="chunk size")),
        # additions (not in the reference)
        ("--target_path", dict(type=str, default=None, help="local HF checkpoint dir of the target")),
        ("--draft_path", dict(type=str, default=None, help="local HF checkpoint dir of the draft")),
        ("--seed", dict(type=int, default=0)),
        ("--kv_dtype", dict(type=str, default="fp16", choices=["fp16", "e4m3"],
                            help="full-KV store: fp16, or FP8 E4M3 with a per-row power-of-two scale (changes the target's numerics)")),
        ("--weight_dtype", dict(type=str, default="fp16", choices=["fp16", "e4m3"],
                                help="target projection weights: fp16, or FP8 E4M3 with a per-row power-of-two scale "
                                     "(changes the target's numerics)")),
    ],
    "offloading_TP": _COMMON_TP_FLAGS + [("--gamma", dict(type=str, default=6))],
    "offloading_seqouia": _COMMON_TP_FLAGS + [("--tree_size", dict(type=str, default="512"))],
}

# the hub ids the reference maps its `--target` names to (offloading_TP.py:52-61); resolved to shapes by triforce_b200.tp
HUB_NAMES = {
    "llama-13B-128K": "NousResearch/Yarn-Llama-2-13b-128k",
    "llama-7B-128K": "NousResearch/Yarn-Llama-2-7b-128k",
    "lwm-128K": "LargeWorldModel/LWM-Text-Chat-128K",
    "lwm-128K-base": "LargeWorldModel/LWM-Text-128K",
}


def build_parser(entry: str) -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="args for main.py")
    for flag, kw in FLAGS[entry]:
        parser.add_argument(flag, **kw)
    return parser


class SyntheticTokenizer:
    """Stands in for AutoTokenizer offline: the loops only read `eos_token_id` and call `decode`."""
    eos_token_id = 2

    def decode(self, *a, **k):
        return ""


def synthetic_prompts(vocab_size: int, prefill: int, seed: int) -> List[torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab_size, (1, prefill), generator=g)]


def _hub_name(target: str) -> str:
    if target not in HUB_NAMES:
        raise NotImplementedError(target)
    return HUB_NAMES[target]


def _finish_distributed():
    import torch.distributed as dist

    dist.barrier()
    sys.stdout.flush()
    os._exit(0)  # NCCL communicators captured in CUDA graphs can stall interpreter teardown


# ---------------------------------------------------------------------------------------------------------------------
# test/on_chip.py
# ---------------------------------------------------------------------------------------------------------------------
def run_on_chip(argv: Optional[List[str]] = None) -> None:
    """AR baseline, TriForce warm-ups, timed TriForce, latency / acceptance / speed-up report (on_chip.py:46-124)."""
    from .cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from .decoding import Autoregressive, TriForce
    from .engine import GraphInferenceEngine
    from .hf_compat import DraftLlamaForCausalLM, TargetLlamaForCausalLM
    from .misc import print_config

    args = build_parser("on_chip").parse_args(argv)
    torch.manual_seed(args.seed)  # the reference never seeds on_chip.py; a parity run needs it (SURVEY §4)
    if args.target != "llama-7B-128K":
        raise NotImplementedError(args.target)
    # no checkpoints offline: a hub id means seeded random-init weights of that architecture, stated explicitly (and printed)
    tpath, dpath = args.target_path or HUB_NAMES[args.target], args.draft_path or "JackFram/llama-68m"
    target = TargetLlamaForCausalLM.from_pretrained(tpath, torch_dtype=torch.float16, device_map="cuda:0", seed=1,
                                                    synthetic=not os.path.isdir(tpath), weight_dtype=args.weight_dtype).eval()
    draft = DraftLlamaForCausalLM.from_pretrained(dpath, torch_dtype=torch.float16, device_map="cuda:0", seed=2,
                                                  synthetic=not os.path.isdir(dpath)).eval()
    tokenizer = SyntheticTokenizer()
    prompts = synthetic_prompts(target.config.vocab_size, args.prefill, args.seed)
    top_k, top_p, temperature = -1, args.top_p, args.temp
    prefill, gen_len, gamma = args.prefill, args.gen_len, args.gamma
    print_config(draft, target, prefill, gen_len, gamma, top_k, top_p, temperature, file_path=None, method="TriForce",
                 spec_args={"budget": args.budget, "chunk_size": args.chunk_size}, dataset=args.dataset)

    # caches and engine (on_chip.py:76-83)
    cache = FlashSimpleCache(target, prefill + gen_len + 16, kv_dtype=args.kv_dtype)
    graph_cache = RetrievalCache(target, max_budget=args.budget, prefill=prefill, gamma=gamma, chunk_size=args.chunk_size)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=args.draft_cache_budget - 16 - gamma, gamma=gamma)
    engine = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    engine.initialize_cuda_graph(gamma, probs=True, temperature=temperature, top_p=top_p)
    for c in (cache, graph_cache, draft_cache):
        c.print_status()
    print(f"tokenized_prompts length: {len(prompts)}")

    def on_device(p):
        return p.to(target.device)[:, :prefill]

    def autoregressive(ids):
        return Autoregressive(tokenizer, engine, ids, max_len=gen_len, top_k=top_k, top_p=top_p, temperature=temperature,
                              verbose=args.verbose)

    def triforce(ids):
        return TriForce(tokenizer, engine, ids, gamma=gamma, max_len=gen_len, top_k=top_k, top_p=top_p, temperature=temperature,
                        verbose=args.verbose, file_path=None, dataset=args.dataset)

    autoregressive(on_device(prompts[0]))                               # 1 warm-up (on_chip.py:91-94)
    ar_speeds = [autoregressive(on_device(p)) for p in prompts[:1]]
    baseline_latency = 1000 / (sum(ar_speeds) / len(ar_speeds))
    print(f"[Autoregressive] average latency: {baseline_latency} ms")

    for _ in range(3):                                                  # 3 warm-ups (on_chip.py:104-107)
        triforce(on_device(prompts[0]))
    results = [triforce(on_device(p)) for p in prompts]
    acceptance = [r[0] for r in results]
    speeds = [r[1] for r in results]
    method_latency = 1000 / (sum(speeds) / len(speeds))
    print(f"average acceptance rate (NOT per token): {sum(acceptance) / len(acceptance)}")
    print(f"[TriForce] average latency: {method_latency} ms")
    print(f"[E2E Speedup]: {baseline_latency / method_latency}")


# ---------------------------------------------------------------------------------------------------------------------
# test/offloading_TP.py and test/offloading_seqouia.py (one process per GPU under torchrun)
# ---------------------------------------------------------------------------------------------------------------------
def _tp_setup(entry: str, argv):
    from .tp import distributed_init

    args = build_parser(entry).parse_args(argv)  # before the rendezvous, so that --help works outside torchrun
    local_rank, world_size = distributed_init()
    device = torch.device("cuda", local_rank)
    torch.manual_seed(args.seed)
    return args, local_rank, world_size, device, _hub_name(args.target)


def _tp_baseline(args, hub, local_rank, world_size, device, input_ids):
    """`--baseline`: the autoregressive TP loop (offloading_TP.py:75-86, offloading_seqouia.py:94-106)."""
    import torch.distributed as dist

    from .decoding import Baseline_Dist
    from .synth import cuda_state_dict
    from .tp import DistributedLlama

    llm = DistributedLlama(model_name_or_path=hub, local_rank=local_rank, world_size=world_size, prefill=args.prefill,
                           gen_len=args.gen_len, temperature=args.temp, top_p=args.top_p, flash_attn=True, retrieval_budget=0,
                           kv_offload=True, on_chip_layers=args.on_chip)
    llm.init_parameters(state_dict=cuda_state_dict(llm.config, seed=1, device=device), cuda_graphs=False)
    latency_ms, _ = Baseline_Dist(SyntheticTokenizer(), llm, input_ids, max_len=args.gen_len, temperature=args.temp,
                                  top_p=args.top_p, local_rank=local_rank)
    if local_rank == 0:
        print(f"\n[Autoregressive] average latency: {latency_ms / 1000} s")
    dist.barrier()


def run_offloading_tp(argv: Optional[List[str]] = None) -> None:
    """TriForce with the target head-sharded over the ranks (offloading_TP.py:88-121)."""
    from .cache import StreamingLLMEvictionCache
    from .decoding import TriForce_Dist
    from .hf_compat import DraftLlamaForCausalLM
    from .synth import cuda_state_dict
    from .tp import DistributedLlama

    args, local_rank, world_size, device, hub = _tp_setup("offloading_TP", argv)
    prompts = [p.to(device) for p in synthetic_prompts(32000, args.prefill, args.seed)]
    if args.baseline:
        _tp_baseline(args, hub, local_rank, world_size, device, prompts[0])
        _finish_distributed()
    gamma = int(args.gamma)
    draft = DraftLlamaForCausalLM.from_pretrained("JackFram/llama-68m", torch_dtype=torch.float16, device_map=device, seed=2, synthetic=True)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    llm = DistributedLlama(model_name_or_path=hub, local_rank=local_rank, world_size=world_size, prefill=args.prefill,
                           gen_len=args.gen_len, temperature=args.temp, top_p=args.top_p, flash_attn=True,
                           retrieval_budget=args.budget, kv_offload=True, on_chip_layers=args.on_chip, draft=draft,
                           draft_cache=draft_cache, gamma=gamma)
    llm.init_parameters(state_dict=cuda_state_dict(llm.config, seed=1, device=device))
    tokens, latencies = [], []
    for ids in prompts:
        avg_tokens, latency = TriForce_Dist(SyntheticTokenizer(), llm, ids[:, :args.prefill], gamma=gamma, max_len=args.gen_len,
                                            top_k=-1, top_p=args.top_p, temperature=args.temp, verbose=False, file_path=None,
                                            dataset=args.dataset)
        tokens.append(avg_tokens)
        latencies.append(latency)
        if local_rank == 0:
            print(f"\n[TriForce] average latency: {latency} s")
            print(f"[TriForce] average accepted tokens: {avg_tokens}")
    if local_rank == 0:
        print(f"[Overall Latency]: {np.array(latencies).mean()}")
        print(f"[Overall Avg Accepted Tokens]: {np.array(tokens).mean()}")
    _finish_distributed()


def run_offloading_seqouia(argv: Optional[List[str]] = None) -> None:
    """TriForce with a Sequoia tree (offloading_seqouia.py:108-207): the tree is grown over the retrieval cache
    (`SpecTree.construct_grow_map`), verified in one masked pass over the full KV (`SpecTree.verify`), and the accepted
    nodes' KV rows are compacted in place.  The grow map is the reference's `tree/512.pt` re-encoded as
    `triforce_b200/data/tree_512.json`; the per-level sampling-without-replacement callables and gather indices of the
    script (:119-133) are built inside SpecTree from it."""
    import torch.distributed as dist

    from .spectree import SpecTree, get_residual, load_grow_map
    from .synth import cuda_state_dict
    from .tp import DistributedLlama

    args, local_rank, world_size, device, hub = _tp_setup("offloading_seqouia", argv)
    grow_map = load_grow_map(args.tree_size)  # reference: torch.load(f'tree/{args.tree_size}.pt')
    prompts = synthetic_prompts(32000, args.prefill, args.seed)
    if args.baseline:
        _tp_baseline(args, hub, local_rank, world_size, device, prompts[0][:, :args.prefill].to(device))
        _finish_distributed()
    llm = DistributedLlama(model_name_or_path=hub, local_rank=local_rank, world_size=world_size, prefill=args.prefill,
                           gen_len=args.gen_len, temperature=args.temp, top_p=args.top_p, flash_attn=True,
                           retrieval_budget=args.budget, kv_offload=True, on_chip_layers=args.on_chip, tree_size=grow_map["size"])
    llm.init_parameters(state_dict=cuda_state_dict(llm.config, seed=1, device=device), cuda_graphs=False)
    tree = SpecTree(engine=llm, temperature=args.temp, top_p=args.top_p, max_length=args.prefill + args.gen_len, grow_map=grow_map,
                    residual_graph=get_residual, tokenizer=SyntheticTokenizer(), vocab_size=llm.config.vocab_size)
    latencies, accepted = [], []
    for prompt in prompts:
        ids = prompt[0, :args.prefill].to(llm.device)
        with torch.inference_mode():
            n, counts = 0, []
            next_token = tree.prefill(prefix=ids)
            torch.cuda.synchronize()
            t0 = time.time()
            while n < args.gen_len:
                tree.construct_grow_map(next_token=next_token)
                next_token, acc_count, _ = tree.verify()
                if next_token is None:  # EOS accepted
                    break
                next_token = next_token.unsqueeze(0)
                n += acc_count
                counts.append(acc_count)
            if n < 64:  # offloading_seqouia.py:191-192: too short to report
                continue
            torch.cuda.synchronize()
            per_token = (time.time() - t0) / n
            dist.barrier()
            if local_rank == 0:
                print(f"[Avg Accepted Tokens]: {np.array(counts).mean()}")
                print(f"[TriForce] average latency: {per_token} s ({n})")
            latencies.append(per_token)
            accepted.append(np.array(counts).mean())
    if local_rank == 0 and latencies:
        print(f"[Overall Latency]: {np.array(latencies).mean()}")
        print(f"[Overall Avg Accepted Tokens]: {np.array(accepted).mean()}")
    _finish_distributed()
