"""Log-likelihood of one document under the target, per store and weight format.

The document (token ids: synthetic from --seed, or an .npy file of ids the user tokenized) is prefilled with
`LlamaModel.prefill(..., logprobs=...)` once per format leg: fp16 weights over an fp16 store ("fp16"), an E4M3 full-KV store
("kv_e4m3"), E4M3 projection weights ("w_e4m3") and both ("both").  Every leg runs in a subprocess of its own on the same ids
and writes its per-position arrays (`logprobs` fp32 [N-1]: log p(ids[i+1] | ids[:i+1]); `argmax` int32 [N-1]) to
`--out/<leg>.npz`.  The leg also times the prefill without scoring on the same reset store: after one untimed scored prefill
(which runs every shape both variants use), it alternates unscored and scored prefills `--repeats` times each, the order
swapped every repeat, and reports the mean, the spread and the paired differences.  Every scored repeat must give the same
bits.  A prefill over an E4M3 store scores exactly what fp16 scores: the prompt attends over an fp16 scratch and the store
is read only afterwards, so the store's cost shows in later turns (`Session.score`), not here.

Printed (one JSON line): per leg the perplexity exp(-mean logprob), the mean and max |delta logprob| against the fp16 leg, the
share of positions whose argmax differs from the fp16 leg's, prefill seconds with and without scoring (mean, standard
deviation, every repeat) and the overhead of scoring (the mean and spread of the paired differences), and the card's name and
power limit.  With synthetic weights (the default: random-init weights from --weight-seed) these numbers show that the tool
works, not what quality a real model keeps; the output says so.

    python tools/perplexity.py [--tokens 124928] [--ids doc.npy] [--legs fp16,kv_e4m3,w_e4m3,both] [--out DIR]
    python tools/perplexity.py --dry-run          # argument checks and the memory arithmetic, no GPU
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LEGS = {"fp16": ("fp16", "fp16"), "kv_e4m3": ("e4m3", "fp16"), "w_e4m3": ("fp16", "e4m3"), "both": ("e4m3", "e4m3")}  # (kv, weights)
SYNTHETIC_NOTE = ("synthetic random-init weights: these numbers show that the tool works, not what quality a real model keeps "
                  "in each format")


def parse_args(argv=None) -> argparse.Namespace:
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--model", default="llama-7B-128K", help="named model shape (triforce_b200.config.named_config)")
    p.add_argument("--layers", type=int, default=0, help="decoder layers (0: the shape's own)")
    p.add_argument("--tokens", type=int, default=124928, help="document length of the synthetic ids")
    p.add_argument("--ids", default=None, help=".npy file of token ids (1-D or [1, N]); replaces the synthetic ids")
    p.add_argument("--seed", type=int, default=0, help="seed of the synthetic ids")
    p.add_argument("--weight-seed", type=int, default=1, help="seed of the synthetic weights")
    p.add_argument("--chunk", type=int, default=128, help="prefill piece length")
    p.add_argument("--repeats", type=int, default=3, help="timed prefills of each variant (without / with scoring) per leg")
    p.add_argument("--legs", default=",".join(LEGS), help=f"comma-separated subset of {','.join(LEGS)}")
    p.add_argument("--out", default="perplexity_out", help="directory of the per-position arrays")
    p.add_argument("--dry-run", action="store_true", help="check the arguments and print the shape arithmetic; no GPU")
    p.add_argument("--leg", default=None, help=argparse.SUPPRESS)  # one leg, in the subprocess
    a = p.parse_args(argv)
    a.legs = [x for x in a.legs.split(",") if x]
    bad = [x for x in a.legs if x not in LEGS]
    if bad or not a.legs:
        p.error(f"--legs: unknown leg(s) {bad}; choose from {list(LEGS)}")
    if a.tokens < 2 and a.ids is None:
        p.error("--tokens: a document needs at least two ids")
    if a.chunk < 1 or a.layers < 0 or a.repeats < 1:
        p.error("--chunk and --repeats must be >= 1 and --layers >= 0")
    return a


def model_config(a):
    import dataclasses

    from triforce_b200.config import named_config
    cfg = named_config(a.model)
    return dataclasses.replace(cfg, num_hidden_layers=a.layers) if a.layers else cfg


def load_ids(a, vocab: int) -> np.ndarray:
    """The document's ids, int64 [N], checked against the vocabulary."""
    if a.ids is not None:
        ids = np.load(a.ids).reshape(-1).astype(np.int64)
    else:
        ids = np.random.default_rng(a.seed).integers(0, vocab, size=a.tokens, dtype=np.int64)
    if ids.size < 2:
        raise SystemExit(f"{a.ids}: a document needs at least two ids, got {ids.size}")
    if ids.min() < 0 or ids.max() >= vocab:
        raise SystemExit(f"token ids must lie in [0, {vocab}); got [{ids.min()}, {ids.max()}]")
    return ids


def shape_arithmetic(N: int, cfg, chunk: int) -> dict:
    """What scoring adds to a prefill of N ids, from shapes: the logits the kernel reads (fp32, every row but the last), the
    lm_head FLOPs the layer-major legs add (every piece but the last), the per-piece buffers, and the fp32 logits of the whole
    document that piece-wise reduction avoids holding."""
    V, h = cfg.vocab_size, cfg.hidden_size
    pieces = -(-N // chunk)
    last = N - (pieces - 1) * chunk
    return {"ids": N, "scored_positions": N - 1, "pieces": pieces, "last_piece_rows": last,
            "logits_read_gb": round((N - 1) * V * 4 / 1e9, 3),
            "layer_major_head_tflop": round(2 * (N - last) * h * V / 1e12, 3),
            "piece_logits_mb": round(min(chunk, N) * V * 4 / 1e6, 3),
            "output_arrays_mb": round((N - 1) * 8 / 1e6, 3),
            "whole_document_fp32_logits_gb": round(N * V * 4 / 1e9, 3)}


def card() -> dict:
    import torch
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        info["power_limit_w"] = float(out.strip().splitlines()[0])
    except Exception as e:  # the numbers still stand; say why the limit is missing
        info["power_limit_error"] = repr(e)
    return info


def spread(xs) -> dict:
    """Mean, sample standard deviation and every value of a list of seconds."""
    m = sum(xs) / len(xs)
    sd = (sum((x - m) ** 2 for x in xs) / (len(xs) - 1)) ** 0.5 if len(xs) > 1 else 0.0
    return {"mean_s": round(m, 4), "std_s": round(sd, 4), "all_s": [round(x, 4) for x in xs]}


def run_leg(a) -> dict:
    """One format leg on the GPU: one untimed scored prefill, then unscored and scored prefills alternated (see the module
    docstring); the arrays go to --out/<leg>.npz."""
    import torch

    from triforce_b200.cache import FlashSimpleCache
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import cuda_state_dict

    kv_dtype, weight_dtype = LEGS[a.leg]
    dev = torch.device("cuda", 0)
    cfg = model_config(a)
    ids = torch.from_numpy(np.load(os.path.join(a.out, "ids.npy"))).to(dev)
    N = ids.numel()
    sd = cuda_state_dict(cfg, seed=a.weight_seed, device=dev)
    model = LlamaModel(cfg, sd, device=dev, weight_dtype=weight_dtype)
    del sd
    torch.cuda.empty_cache()
    kv = FlashSimpleCache(model, N + 64, kv_dtype=kv_dtype)
    lp = torch.empty(N - 1, dtype=torch.float32, device=dev)
    am = torch.empty(N - 1, dtype=torch.int32, device=dev)
    times = {False: [], True: []}

    def prefill(scored: bool) -> float:
        kv.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.prefill(ids, kv, chunk=a.chunk, logprobs=(lp, am) if scored else None)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    with torch.inference_mode():
        prefill(True)  # warm-up: module loads, GEMM algorithm choice, allocator growth
        first = (lp.clone(), am.clone())
        for r in range(a.repeats):
            for scored in ((False, True) if r % 2 == 0 else (True, False)):
                times[scored].append(prefill(scored))
                if scored and not (torch.equal(lp, first[0]) and torch.equal(am, first[1])):
                    raise SystemExit(f"leg {a.leg}: a scored prefill repeat gave different scores")
    np.savez(os.path.join(a.out, f"{a.leg}.npz"), logprobs=lp.cpu().numpy(), argmax=am.cpu().numpy())
    diffs = [w - wo for w, wo in zip(times[True], times[False])]
    return {"leg": a.leg, "kv_dtype": kv_dtype, "weight_dtype": weight_dtype, "repeats": a.repeats,
            "prefill_without_scoring": spread(times[False]), "prefill_with_scoring": spread(times[True]),
            "scoring_overhead": spread(diffs), "peak_memory_gb": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2),
            "card": card()}


def summarize(out_dir: str, legs, ids: np.ndarray) -> dict:
    """Perplexity of each leg and its differences from the fp16 leg (when it ran)."""
    arrays = {leg: np.load(os.path.join(out_dir, f"{leg}.npz")) for leg in legs}
    ref = arrays.get("fp16")
    res = {}
    for leg, z in arrays.items():
        lp = z["logprobs"].astype(np.float64)
        r = {"perplexity": float(np.exp(-lp.mean())), "mean_logprob": float(lp.mean()),
             "greedy_share": float((z["argmax"] == ids[1:]).mean())}
        if ref is not None and leg != "fp16":
            d = np.abs(lp - ref["logprobs"].astype(np.float64))
            r.update(mean_abs_delta_logprob=float(d.mean()), max_abs_delta_logprob=float(d.max()),
                     argmax_differs_share=float((z["argmax"] != ref["argmax"]).mean()))
        res[leg] = r
    return res


def main(argv=None) -> int:
    a = parse_args(argv)
    cfg = model_config(a)
    if a.leg is not None:
        print(json.dumps(run_leg(a)), flush=True)
        return 0
    ids = load_ids(a, cfg.vocab_size)
    arith = shape_arithmetic(ids.size, cfg, a.chunk)
    if a.dry_run:
        print(json.dumps({"dry_run": True, "model": a.model, "layers": cfg.num_hidden_layers, "legs": a.legs, "out": a.out,
                          "shapes": arith}))
        return 0
    os.makedirs(a.out, exist_ok=True)
    np.save(os.path.join(a.out, "ids.npy"), ids)
    child = [sys.executable, os.path.abspath(__file__), "--model", a.model, "--layers", str(a.layers), "--chunk", str(a.chunk),
             "--weight-seed", str(a.weight_seed), "--repeats", str(a.repeats), "--out", a.out, "--legs", ",".join(a.legs)]
    runs = {}
    for leg in a.legs:
        p = subprocess.run(child + ["--leg", leg], capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise SystemExit(f"leg {leg} failed (exit {p.returncode})")
        runs[leg] = json.loads(p.stdout.strip().splitlines()[-1])
    quality = summarize(a.out, a.legs, ids)
    for leg in a.legs:
        runs[leg].update(quality[leg])
    print(json.dumps({"model": a.model, "layers": cfg.num_hidden_layers, "ids": "file " + a.ids if a.ids else f"synthetic seed {a.seed}",
                      "weights": SYNTHETIC_NOTE, "shapes": arith, "legs": runs}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
