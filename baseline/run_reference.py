#!/usr/bin/env python
"""MEASUREMENT INFRASTRUCTURE — not product code.  Runs the UNMODIFIED reference (Infini-AI-Lab/TriForce) for timing.

The reference is a script tree (`models/ utils/ test/`, no setup.py), so there is nothing to pip-install: `__graft_entry__.build()`
stages its Python files into the git-ignored `oracle/_ref/` (oracle/stage_ref.py; they never enter the history), and this runner
imports them from there (or from $TRIFORCE_REFERENCE_ROOT).  It
re-creates `test/on_chip.py:76-117` — caches, `GraphInferenceEngine`, `Autoregressive`, `TriForce` — around random-init models
of the benchmark's shapes (there are no checkpoints or tokenizers offline), under the documented shims of SURVEY §8c:

  1. stub `termcolor` (missing; utils/misc.py:2);
  2. `models.modeling_llama.apply_rotary_pos_emb` := the reference's own 4.37-style copy in models/tensor_op.py:25-50
     (transformers 5.5 dropped the `position_ids` argument of the call at modeling_llama.py:222);
  3. plain-RoPE targets only: `_init_rope` takes the reference's own `LlamaRotaryEmbedding` branch (transformers 5.5 never
     leaves `config.rope_scaling` None);
  4. `time.time()` inside utils/decoding.py synchronises the device first (the reference's timed regions, decoding.py:29,36,69,
     143, omit it — SURVEY §8d asks for the synchronised number).

Two modes, one JSON line on stdout:

  --device cuda   the GPU-side comparison bar of SURVEY §8(d): the reference with REAL flash-attn 2.8.3 (`flash_attn_with_kvcache`,
                  where installed) and its own CUDA graphs on the same GPU, same shapes, same seeded weights as bench.py:
                  `Autoregressive` ms/token and `TriForce` tokens/s, each through the reference's own functions (which prefill
                  the whole prompt themselves, untimed, in 128-token chunks).
  --device cpu    the reference's CPU HF-eager path on the host cores (north_star's reported baseline; `bench.py --impl
                  reference`): fp32 weights (the fastest dtype torch's CPU GEMM has), fp16 KV store as the reference allocates it,
                  torch's fused CPU attention in place of flash-attn (no CPU build exists), eager callables in place of CUDA graphs,
                  `torch.Tensor.cuda` a no-op.  Bounded sample: the 124 928-token prompt is NOT prefilled on the CPU (≈ 1.7 PFLOP,
                  hours) — the full KV store is filled with synthetic N(0,1) keys/values, the retrieval cache is then built by the
                  reference's own `init_graph_cache`, the draft window is prefilled from the last 512 prompt tokens; after that
                  exactly W + K outer iterations of the reference's own `TriForce` loop run and the K are timed
                  (`Middle_Spec` entry to `Middle_Spec` entry, tokens from `kv_cache.seq_len`).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)

SHAPES = {  # the checkpoints the reference's entry points load (test/on_chip.py:48-53) — config.json values
    "llama-7B-128K": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                          max_position_embeddings=131072, rms_norm_eps=1e-5,
                          rope_scaling={"type": "yarn", "factor": 32.0, "original_max_position_embeddings": 4096}),
    "llama-13B-128K": dict(hidden_size=5120, intermediate_size=13824, num_hidden_layers=40, num_attention_heads=40,
                           max_position_embeddings=131072, rms_norm_eps=1e-5,
                           rope_scaling={"type": "yarn", "factor": 32.0, "original_max_position_embeddings": 4096}),
    "lwm-128K": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                     max_position_embeddings=131072, rms_norm_eps=1e-5, rope_theta=10000000.0),
    "tiny-yarn-target": dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                             max_position_embeddings=4096, rms_norm_eps=1e-6,
                             rope_scaling={"type": "yarn", "factor": 2.0, "original_max_position_embeddings": 2048}),
    "llama-68M": dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                      max_position_embeddings=2048, rms_norm_eps=1e-6),
}


def reference_root() -> str:
    for cand in (os.environ.get("TRIFORCE_REFERENCE_ROOT"), os.path.join(REPO, "oracle", "_ref")):
        if cand and os.path.isfile(os.path.join(cand, "utils", "decoding.py")) and os.path.isfile(os.path.join(cand, "models", "cache.py")):
            return cand
    raise FileNotFoundError("reference tree not found (oracle/_ref is staged by __graft_entry__.build() where the reference exists)")


def load_reference(root: str, cpu: bool):
    """Import the reference's modules with this repo's same-named drop-in packages (`models`, `utils`) hidden."""
    import torch

    for name in list(sys.modules):
        if name in ("models", "utils", "data") or name.startswith(("models.", "utils.", "data.")):
            del sys.modules[name]
    hidden = {os.path.abspath(REPO), os.path.abspath(os.getcwd())}
    saved = list(sys.path)
    sys.path[:] = [root] + [p for p in sys.path if os.path.abspath(p or os.getcwd()) not in hidden]
    tc = types.ModuleType("termcolor")
    tc.colored = lambda s, *a, **k: s
    sys.modules.setdefault("termcolor", tc)  # shim 1
    try:
        import models.cache as cache
        import models.modeling_llama as ml
        import models.modeling_llama_68m as ms
        import models.tensor_op as top
        import utils.decoding as decoding
        import utils.graph_infer as graph_infer
        import utils.sampling as sampling
        from models.config_yarn import LlamaConfig
    finally:
        sys.path[:] = [root] + [p for p in saved if p != root]
    assert os.path.abspath(ml.__file__).startswith(os.path.abspath(root)), ml.__file__
    ml.apply_rotary_pos_emb = top.apply_rotary_pos_emb  # shim 2
    if cpu:
        ml.flash_attn_with_kvcache = ms.flash_attn_with_kvcache = top.flash_attn_with_kvcache = eager_attention
        torch.Tensor.cuda = lambda self, *a, **k: self
    return types.SimpleNamespace(cache=cache, ml=ml, ms=ms, top=top, decoding=decoding, graph_infer=graph_infer, sampling=sampling,
                                 LlamaConfig=LlamaConfig)


def eager_attention(q, k_cache, v_cache, softmax_scale=None, causal=False, **kw):
    """CPU stand-in for `flash_attn_with_kvcache` (q [b,sq,h,d], k/v [b,sk,h,d], bottom-right causal; flash-attn has no CPU
    build): torch's own fused CPU attention (`scaled_dot_product_attention`, fp32 softmax and accumulation) on the fp16 KV store
    as it lies — measured 6x faster here than the bmm / softmax / bmm formulation of HF's eager path (which converts the whole
    KV to fp32 first), i.e. the choice favours the CPU number."""
    import torch
    import torch.nn.functional as F

    b, sq, h, d = q.shape
    sk = k_cache.shape[1]
    mask = None
    if causal and sq > 1:
        i = torch.arange(sq)[:, None]
        j = torch.arange(sk)[None, :]
        mask = j <= i + sk - sq
    dt = k_cache.dtype
    o = F.scaled_dot_product_attention(q.transpose(1, 2).to(dt), k_cache.transpose(1, 2), v_cache.transpose(1, 2).to(dt), attn_mask=mask,
                                       scale=float(softmax_scale))
    return o.transpose(1, 2).to(q.dtype)


class TokenizerStub:
    eos_token_id = 2

    def decode(self, *a, **k):
        return ""


def build_models(ref, args, device, dtype):
    """Reference model classes, random-init.  cuda: the very weights bench.py uses (triforce_b200.synth.cuda_state_dict seeds 1 / 2);
    cpu: a seeded N(0, 0.02) block tiled over the parameters (27 GB of fp32 — values only steer which tokens are drawn)."""
    import torch
    try:
        from transformers.initialization import no_init_weights
    except ImportError:
        from transformers.modeling_utils import no_init_weights

    cfg_t = ref.LlamaConfig(vocab_size=32000, **SHAPES[args.target])
    cfg_d = ref.LlamaConfig(vocab_size=32000, **SHAPES["llama-68M"])
    # built in fp32 (rotary tables computed in fp32, then cast with the model — as the golden fixtures' models were), on the
    # target device directly, without HF's random init (the weights are overwritten below)
    plain = "rope_scaling" not in SHAPES[args.target]
    if plain:  # shim 3: the reference's own first branch of _init_rope (modeling_llama.py:180-198) for plain-RoPE targets
        attn_cls = ref.ml.LlamaAttention
        orig_init_rope = attn_cls._init_rope
        theta = float(SHAPES[args.target].get("rope_theta", 10000.0))
        attn_cls._init_rope = lambda self: setattr(self, "rotary_emb", ref.ml.LlamaRotaryEmbedding(
            self.head_dim, max_position_embeddings=self.max_position_embeddings, base=theta))
    try:
        with no_init_weights(), torch.device(device):
            target = ref.ml.LlamaForCausalLM(cfg_t).eval()
            draft = ref.ms.LlamaForCausalLM(cfg_d).eval()
    finally:
        if plain:
            attn_cls._init_rope = orig_init_rope
    if device == "cuda":
        target, draft = target.to(dtype), draft.to(dtype)
    if device == "cuda":
        sys.path.append(REPO)  # after the reference's modules are imported: this repo's `models/` must not shadow them
        from triforce_b200.config import named_config
        from triforce_b200.synth import cuda_state_dict
        for model, name, seed in ((target, args.target, 1), (draft, "llama-68M", 2)):
            sd = cuda_state_dict(named_config(name), seed=seed, device="cuda")
            missing = model.load_state_dict(sd, strict=False)
            assert not [k for k in missing.missing_keys if "rotary" not in k and "inv_freq" not in k], missing.missing_keys
            del sd
    else:
        g = torch.Generator().manual_seed(1)
        block = torch.empty(1 << 24, dtype=torch.float32).normal_(0.0, 0.02, generator=g)
        with torch.no_grad():
            for model in (target, draft):
                for k, (name, p) in enumerate(model.named_parameters()):
                    if p.dim() == 1:
                        p.fill_(1.0)  # RMSNorm weights
                        continue
                    flat, off = p.view(-1), (k * 4099) % (1 << 20)
                    for i in range(0, flat.numel(), block.numel() - off):
                        n = min(block.numel() - off, flat.numel() - i)
                        flat[i:i + n] = block[off:off + n]
    return target.to(dtype), draft.to(dtype)


class SyncTime:
    """shim 4: utils.decoding's `time` — synchronise the device before reading the clock."""

    def __init__(self, cuda):
        self.cuda = cuda

    def time(self):
        if self.cuda:
            import torch
            torch.cuda.synchronize()
        return time.time()

    def __getattr__(self, name):
        return getattr(time, name)


class _EnoughSteps(Exception):
    pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--target", default="llama-7B-128K")
    ap.add_argument("--prefill", type=int, default=124928)
    ap.add_argument("--budget", type=int, default=4096)
    ap.add_argument("--chunk_size", type=int, default=8)
    ap.add_argument("--gamma", type=int, default=6)
    ap.add_argument("--temp", type=float, default=0.6)
    ap.add_argument("--top_p", type=float, default=0.9)
    ap.add_argument("--gen_len", type=int, default=96, help="cuda: tokens of the timed TriForce call")
    ap.add_argument("--ar_len", type=int, default=32, help="cuda: tokens of the timed Autoregressive call")
    ap.add_argument("--warmup_calls", type=int, default=1, help="cuda: untimed TriForce calls first (on_chip.py:106-108 does 3)")
    ap.add_argument("--steps", type=int, default=8, help="cpu: timed outer iterations")
    ap.add_argument("--warmup", type=int, default=1, help="cpu: untimed outer iterations")
    ap.add_argument("--threads", type=int, default=0, help="cpu: torch threads (0 = all host CPUs)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--layers", type=int, default=0, help="debugging only: cut the target to this many layers (0 = the real model)")
    args = ap.parse_args()
    if args.layers:
        SHAPES[args.target] = dict(SHAPES[args.target], num_hidden_layers=args.layers)

    if args.device == "cpu":
        if not args.threads:  # one thread per physical core (hyper-threads only add contention to these bandwidth-bound loops)
            c = os.cpu_count() or 1
            args.threads = c // 2 if c >= 16 else c
        n = args.threads
        for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS"):  # torchrun exports OMP_NUM_THREADS=1: pin the same count at every N
            os.environ[k] = str(n)
    import torch

    cuda = args.device == "cuda"
    if not cuda:
        torch.set_num_threads(args.threads)
    t_start = time.time()

    def stage(msg):
        print(f"[run_reference +{time.time() - t_start:7.1f}s] {msg}", file=sys.stderr, flush=True)

    root = reference_root()
    ref = load_reference(root, cpu=not cuda)
    dec = ref.decoding
    dec.time = SyncTime(cuda)
    dtype = torch.float16 if cuda else torch.float32
    target, draft = build_models(ref, args, args.device, dtype)
    stage("models built")
    P, gamma = args.prefill, args.gamma
    gen_cap = max(args.gen_len, args.ar_len, 8 * (args.steps + args.warmup + 2)) + 64
    cache_model = target
    if not cuda:
        # the reference's caches take their dtype from the weights (cache.py:30,136); the CPU path computes in fp32 but keeps the
        # KV stores fp16 — what the reference holds on the GPU, and half the host memory (66 GB instead of 131 GB)
        w16 = types.SimpleNamespace(weight=torch.empty(0, dtype=torch.float16))
        cache_model = types.SimpleNamespace(config=target.config, device=target.device, model=types.SimpleNamespace(
            layers=[types.SimpleNamespace(self_attn=types.SimpleNamespace(q_proj=w16))]))
    cache = ref.cache.FlashSimpleCache(cache_model, P + gen_cap + 16)
    graph_cache = ref.cache.RetrievalCache(cache_model, max_budget=args.budget, prefill=P, gamma=gamma, chunk_size=args.chunk_size)
    draft_cache = ref.cache.StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = ref.graph_infer.GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    g = torch.Generator().manual_seed(args.seed)
    input_ids = torch.randint(0, 32000, (1, P), generator=g).to(args.device)  # bench.py's prompt
    tok = TokenizerStub()
    out = {"impl": "reference", "device": args.device, "reference_root": os.path.relpath(root, REPO) if root.startswith(REPO) else root,
           "target": args.target, "prefill": P, "budget": args.budget, "chunk_size": args.chunk_size, "gamma": gamma,
           "temperature": args.temp, "top_p": args.top_p, "torch": torch.__version__}
    torch.manual_seed(args.seed)

    if cuda:
        import flash_attn
        out["flash_attn"] = flash_attn.__version__
        out["gpu"] = torch.cuda.get_device_name(0)
        ge.initialize_cuda_graph(gamma, probs=True, temperature=args.temp, top_p=args.top_p)
        t0 = time.time()
        ar_tps = dec.Autoregressive(tok, ge, input_ids, max_len=args.ar_len, top_k=-1, top_p=args.top_p, temperature=args.temp)
        torch.cuda.synchronize()
        out["autoregressive"] = {"tokens_per_s": ar_tps, "ms_per_token": 1000.0 / ar_tps, "tokens": args.ar_len,
                                 "call_seconds_incl_prefill": time.time() - t0,
                                 "how": "utils/decoding.py::Autoregressive (eager full-KV decode, flash_attn_with_kvcache), device-synchronised clock"}
        for _ in range(args.warmup_calls):
            dec.TriForce(tok, ge, input_ids, gamma=gamma, max_len=8, top_k=-1, top_p=args.top_p, temperature=args.temp)
        steps = []
        orig_mid = dec.Middle_Spec

        def mid(*a, **k):
            steps.append(cache.seq_len)
            return orig_mid(*a, **k)

        dec.Middle_Spec = mid
        t0 = time.time()
        acc, tps = dec.TriForce(tok, ge, input_ids, gamma=gamma, max_len=args.gen_len, top_k=-1, top_p=args.top_p, temperature=args.temp)
        torch.cuda.synchronize()
        dec.Middle_Spec = orig_mid
        n_tokens = cache.seq_len - P  # committed tokens of the call (+1 sampled, not yet appended)
        out["triforce"] = {"tokens_per_s": tps, "ms_per_token": 1000.0 / tps, "acceptance_rate": acc, "outer_steps": len(steps),
                           "tokens": n_tokens, "ms_per_step": 1000.0 * (n_tokens / tps) / max(len(steps), 1),
                           "tokens_per_step": n_tokens / max(len(steps), 1), "call_seconds_incl_prefill": time.time() - t0,
                           "how": "utils/decoding.py::TriForce after %d warm-up call(s) (so the draft window runs with the zero sinks of "
                                  "the reference's timed runs), real flash-attn + the reference's CUDA graphs, device-synchronised clock" % args.warmup_calls}
        out["speedup_vs_ar"] = tps / ar_tps
        out["max_memory_gb"] = torch.cuda.max_memory_allocated() / 1e9
    else:
        for gq in range(gamma + 3):  # eager callables in place of the CUDA graphs (graph_infer.py:136-164 needs a GPU)
            ge.callables[gq] = (lambda ids, gq=gq: ge.engine.draft_run(input_ids=ids, gamma_offset=gq, probs=True, temperature=args.temp,
                                                                       top_p=args.top_p))
        ge.callable_model_verify = (lambda ids, pos: ge.engine.model_verify(input_ids=ids, position_ids=pos, probs=True,
                                                                            temperature=args.temp, top_p=args.top_p))
        # synthetic prompt KV (bounded sample): N(0,1) keys and values, tiled from one block
        gk = torch.Generator().manual_seed(7)
        blk = torch.empty((8192, cache.key_cache.shape[-2], cache.key_cache.shape[-1])).normal_(generator=gk).to(torch.float16)
        for l in range(cache.key_cache.shape[0]):
            for s0 in range(0, P, 4096):
                n = min(4096, P - s0)
                ko, vo = (l * 131 + s0 // 4096 * 17) % 4096, (l * 257 + s0 // 4096 * 29 + 1024) % 4096
                cache.key_cache[l, 0, s0:s0 + n] = blk[ko:ko + n]
                cache.value_cache[l, 0, s0:s0 + n] = blk[vo:vo + n]
        stage("synthetic KV store filled")
        # the one dtype seam of the fp32-weights CPU path: the retrieval scoring multiplies q by the fp16 chunk means with
        # torch.matmul (cache.py:157), which needs one dtype — hand it the fp16 query the reference's fp16 model would have
        orig_build = ref.cache.RetrievalCache.init_graph_cache
        ref.cache.RetrievalCache.init_graph_cache = lambda self, kv_cache, query_states, layer_idx: orig_build(
            self, kv_cache, query_states.to(torch.float16), layer_idx)
        orig_inf, orig_dpre, orig_reset, orig_mid = ge.inference, ge.graph_draft_prefill, cache.reset, dec.Middle_Spec

        def inference(input_ids):
            if input_ids.shape[-1] > 64:  # the prompt: already "in" the synthetic KV store
                cache.seq_len = input_ids.shape[-1]
                return None
            return orig_inf(input_ids=input_ids)

        marks = []

        def mid(*a, **k):
            marks.append((time.perf_counter(), cache.seq_len))
            stage(f"outer iteration {len(marks)} starts (kv {cache.seq_len})")
            if len(marks) > args.warmup + args.steps:
                raise _EnoughSteps()
            return orig_mid(*a, **k)

        ge.inference = inference
        ge.graph_draft_prefill = lambda input_ids: orig_dpre(input_ids=input_ids[:, -512:])
        cache.reset = lambda: None  # keep the synthetic store (reset would zero 66 GB and the length)
        dec.Middle_Spec = mid
        out["setup_seconds"] = time.time() - t_start
        try:
            dec.TriForce(tok, ge, input_ids, gamma=gamma, max_len=1 << 30, top_k=-1, top_p=args.top_p, temperature=args.temp)
        except _EnoughSteps:
            pass
        (t0, s0), (t1, s1) = marks[args.warmup], marks[args.warmup + args.steps]
        tokens, secs = s1 - s0, t1 - t0
        out["triforce"] = {"tokens_per_s": tokens / secs, "ms_per_step": 1000.0 * secs / args.steps, "steps": args.steps, "warmup": args.warmup,
                           "tokens": tokens, "tokens_per_step": tokens / args.steps, "seconds": secs,
                           "step_seconds": [round(marks[i + 1][0] - marks[i][0], 3) for i in range(len(marks) - 1)]}
        out["threads"] = torch.get_num_threads()
        out["host_cpus"] = os.cpu_count()
    out["total_seconds"] = time.time() - t_start
    print("REFERENCE_JSON " + json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
