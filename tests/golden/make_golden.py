#!/usr/bin/env python
"""Generates the committed golden fixtures in this directory FROM THE REFERENCE ITSELF (run in the build container,
where /root/reference exists).  Usage:  python tests/golden/make_golden.py

The reference ships no tests or golden vectors (SURVEY.md §4), so these fixtures — outputs of the reference's own
Python (`models/cache.py`, `utils/sampling.py`, `utils/decoding.py`, `models/modeling_llama*.py`) executed on CPU under
the shims documented in `oracle/ref_harness.py` — are what pins `oracle/triforce_oracle.py`.  Inputs are regenerated
from PCG64 seeds by the tests (see `tests/golden_inputs.py`), so only outputs are stored.

Files written:
  retrieval_build.npz   reference RetrievalCache.init_graph_cache: fp16 chunk scores, raw torch.topk indices, cache rows
  sampling.npz          reference norm_logits / max_fn on seeded logits
  forward.npz           reference target forward: last-token logits after a chunked prefill, retrieval-verify logits
  yarn_7b_rows.npz      rows of the reference's YaRN cos/sin tables at the 7B / 13B geometry (see yarn_7b_row_indices)
  e2e_<cfg>.json        event traces (every sample / rand / Middle_Spec return / target input) of TriForce first and
                        second call (the draft-cache reset quirk, SURVEY §7 hard part 3) and of Autoregressive
  ref_*                 the reference's PG-19 loader, tree file and command lines (see make_reference_files)
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

from oracle import ref_harness as rh  # noqa: E402
from oracle import triforce_oracle as orc  # noqa: E402
from triforce_b200.config import named_config  # noqa: E402
from triforce_b200.rng import CounterNoise  # noqa: E402
from triforce_b200.synth import numpy_state_dict, numpy_prompt  # noqa: E402
import golden_inputs as gi  # noqa: E402


class _ShapeModel:
    """Just enough of an HF model for the reference cache constructors (cache.py:25-33,131-139)."""

    def __init__(self, L, H, d):
        self.config = type("C", (), dict(hidden_size=H * d, num_key_value_heads=H, num_attention_heads=H,
                                         num_hidden_layers=L))()
        w = type("W", (), dict(dtype=torch.float16))()
        attn = type("A", (), dict(q_proj=type("Q", (), dict(weight=w))()))()
        self.model = type("M", (), dict(layers=[type("Lyr", (), dict(self_attn=attn))()]))()
        self.device = torch.device("cpu")


def make_retrieval_build():
    ref = rh.load_reference()
    out = {}
    for case in gi.RETRIEVAL_CASES:
        name, H, d, P, chunk, budget, seed = case
        K, V, q = gi.retrieval_inputs(case)
        m = _ShapeModel(1, H, d)
        kv = ref.cache.FlashSimpleCache(m, P + 8)
        kv.key_cache[0, 0, :P] = torch.from_numpy(K)
        kv.value_cache[0, 0, :P] = torch.from_numpy(V)
        kv.seq_len = P
        rc = ref.cache.RetrievalCache(m, max_budget=budget, prefill=P, chunk_size=chunk, gamma=4)
        rec = {}
        orig_torch = ref.cache.torch

        class _Proxy:
            def __getattr__(self, n):
                return getattr(orig_torch, n)

            @staticmethod
            def topk(x, k, dim=-1, **kw):
                v, i = orig_torch.topk(x, k=k, dim=dim, **kw)
                rec["scores_rest"] = x.clone()
                rec["idx_rest"] = i.clone()
                return v, i

        ref.cache.torch = _Proxy()
        try:
            rc.init_graph_cache(kv, torch.from_numpy(q).reshape(1, 1, H, d), 0)
        finally:
            ref.cache.torch = orig_torch
        scores_rest = rec["scores_rest"][0].numpy()  # [H, chunks-1] fp16 (chunk 0 excluded by the reference slice)
        idx = rec["idx_rest"][0].numpy().astype(np.int32) + 1  # raw torch.topk order, shifted like cache.py:160
        out[f"{name}.scores_rest"] = scores_rest
        out[f"{name}.topk_idx_rest"] = idx
        rk = rc.key_cache[0, 0, :budget].numpy()
        rv = rc.value_cache[0, 0, :budget].numpy()
        # store a digest of the gathered rows instead of megabytes: per-(slot-chunk, head) sums in fp64
        out[f"{name}.retrK_digest"] = rk.astype(np.float64).reshape(budget // chunk, chunk, H, d).sum((1, 3))
        out[f"{name}.retrV_digest"] = rv.astype(np.float64).reshape(budget // chunk, chunk, H, d).sum((1, 3))
        # cross-check the oracle while we are here
        oK, oV, oidx, osc = orc.retrieval_build(K, V, q, P, chunk, budget)
        ulp_diff = (osc[:, 1:].view(np.int16).astype(np.int32) - scores_rest.view(np.int16).astype(np.int32))
        frac = float((ulp_diff != 0).mean())
        same_set = all(set(oidx[h, 1:]) == set(idx[h]) for h in range(H))
        print(f"[retrieval_build:{name}] oracle-vs-reference score mismatch frac={frac:.5f} "
              f"max|ulp|={np.abs(ulp_diff).max()} same top-k set={same_set}")
        out[f"{name}.oracle_score_mismatch_frac"] = np.float64(frac)
    np.savez_compressed(os.path.join(HERE, "retrieval_build.npz"), **out)


def make_sampling():
    ref = rh.load_reference()
    out = {}
    for case in gi.SAMPLING_CASES:
        name = case[0]
        logits = gi.sampling_logits(case)
        T, top_p = case[4], case[5]
        probs = ref.sampling.norm_logits(torch.from_numpy(logits.copy()), temperature=T, top_k=-1, top_p=top_p).numpy()
        out[f"{name}.probs"] = probs.astype(np.float32)
        o = orc.norm_logits(logits.copy(), T, -1, top_p)
        print(f"[sampling:{name}] kept ref={int((probs > 0).sum())} oracle={int((o > 0).sum())} "
              f"mask mismatches={int(((probs > 0) != (o > 0)).sum())} max|dp|={np.abs(o - probs).max():.3e}")
        p, q = gi.residual_pair(case)
        out[f"{name}.max_fn"] = ref.sampling.max_fn(torch.from_numpy(p - q)).numpy()
    np.savez_compressed(os.path.join(HERE, "sampling.npz"), **out)


def _models(case):
    ts, ds = named_config(case["target"]), named_config(case["draft"])
    tsd = numpy_state_dict(ts, case["target_seed"])
    dsd = numpy_state_dict(ds, case["draft_seed"])
    target, draft = rh.build_reference_models(ts, ds, tsd, dsd)
    return ts, ds, tsd, dsd, target, draft


def make_forward():
    case = gi.FORWARD_CASE
    ts, ds, tsd, dsd, target, draft = _models(case)
    P, B, c, g = case["prefill"], case["budget"], case["chunk"], case["gamma"]
    ge = rh.build_reference_engine(target, draft, P, 32, B, c, g, case["temperature"], case["top_p"])
    ids = numpy_prompt(P, seed=case["prompt_seed"])
    with torch.inference_mode():
        ge.engine.kv_cache.reset(); ge.engine.graph_cache.reset(); ge.engine.draft_cache.reset()
        ge.inference(input_ids=ids[:, :-1])
        logits_last = ge.inference(input_ids=ids[:, -1:])[0, -1].numpy()
        vt = torch.from_numpy(np.asarray(case["verify_tokens"], dtype=np.int64))[None]
        pos = torch.arange(P, P + g + 1)[None]
        vlogits = ge.engine.model_verify(input_ids=vt, position_ids=pos, probs=False)[0].numpy()
        # full-KV verify of the same rows (non-spec path, graph_cache given but q_len > 1 so no rebuild)
        flogits = ge.inference(input_ids=vt)[0].numpy()
        # draft: prefill then one speculative step of 3 tokens
        ge.graph_draft_prefill(input_ids=ids)
        dlogits = ge.engine.draft_run(input_ids=vt[:, :3], gamma_offset=2, probs=False)[0].numpy()
    rot = target.model.layers[0].self_attn.rotary_emb
    np.savez_compressed(os.path.join(HERE, "forward.npz"),
                        logits_last=logits_last.astype(np.float16), verify_logits=vlogits.astype(np.float16),
                        full_verify_logits=flogits.astype(np.float16), draft_logits=dlogits.astype(np.float16),
                        yarn_cos_rows=rot.cos_cached[:: 97].numpy(), yarn_sin_rows=rot.sin_cached[:: 97].numpy())
    assert np.array_equal(logits_last.astype(np.float16).astype(np.float32), logits_last)
    print("[forward] wrote logits; |logits| max", np.abs(logits_last).max())


YARN_7B_STRIDE = 1021  # strided rows over the whole 131 072-row table


def yarn_7b_row_indices(max_pos: int = 131072) -> np.ndarray:
    """Rows of yarn_7b_rows.npz: every 1021st row, every row of 124 900..124 999 (around the cfg2 prompt end, where fp32
    positions times inv_freq are furthest from exact) and the last 64 rows."""
    rows = np.concatenate([np.arange(0, max_pos, YARN_7B_STRIDE), np.arange(124900, 125000), np.arange(max_pos - 64, max_pos)])
    return np.unique(rows).astype(np.int64)


def make_yarn_7b():
    """The reference's LlamaYaRNRotaryEmbedding at the 7B / 13B geometry (head_dim 128, 131 072 positions, factor 32 over an
    original 4096), built on the CPU as the reference builds it (modeling_llama.py:187-194)."""
    ref = rh.load_reference()
    rot = ref.ml.LlamaYaRNRotaryEmbedding(128, max_position_embeddings=131072, base=10000, scaling_factor=32.0,
                                          original_max_position_embeddings=4096)
    rows = yarn_7b_row_indices()
    np.savez_compressed(os.path.join(HERE, "yarn_7b_rows.npz"), rows=rows, cos=rot.cos_cached[rows].numpy(),
                        sin=rot.sin_cached[rows].numpy())
    print(f"[yarn_7b] wrote {len(rows)} rows of the 131072 x 128 tables")


def make_e2e():
    ref = rh.load_reference()
    tok = rh.TokenizerStub()
    only = os.environ.get("GOLDEN_E2E_ONLY")  # regenerate one case: GOLDEN_E2E_ONLY=plain [GOLDEN_NOISE_SEED=n]
    for case in gi.E2E_CASES:
        if only and case["name"] != only:
            continue
        if os.environ.get("GOLDEN_NOISE_SEED"):
            case = dict(case, noise_seed=int(os.environ["GOLDEN_NOISE_SEED"]))
        t0 = time.time()
        ts, ds, tsd, dsd, target, draft = _models(case)
        P, B, c, g, gen = case["prefill"], case["budget"], case["chunk"], case["gamma"], case["gen_len"]
        T, top_p = case["temperature"], case["top_p"]
        ge = rh.build_reference_engine(target, draft, P, gen + 16, B, c, g, T, top_p)
        ids = numpy_prompt(P, seed=case["prompt_seed"])
        ot = orc.LlamaOracle(ts, {k: v.numpy() for k, v in tsd.items()}, False)
        od = orc.LlamaOracle(ds, {k: v.numpy() for k, v in dsd.items()}, True)
        rot = target.model.layers[0].self_attn.rotary_emb
        rd = draft.model.layers[0].self_attn.rotary_emb
        ot.set_tables(rot.cos_cached.numpy(), rot.sin_cached.numpy())
        od.set_tables(rd.cos_cached.numpy().astype(np.float16), rd.sin_cached.numpy().astype(np.float16))
        eng = orc.EngineOracle(ot, od, P, gen + 16, B, c, g, T, top_p)
        record = dict(case=case, calls=[])
        for call in range(2):
            trace = []
            with rh.traced_random(CounterNoise(case["noise_seed"]), trace), rh.traced_calls(ge, trace):
                acc, _ = ref.decoding.TriForce(tok, ge, ids, gamma=g, max_len=gen, top_k=-1, top_p=top_p, temperature=T)
            res = orc.triforce(eng, ids.numpy(), g, gen, CounterNoise(case["noise_seed"]))
            same = 0
            for a, b in zip(trace, res["trace"]):
                if a[0] != b[0] or a[1] != b[1]:
                    break
                same += 1
            record["calls"].append(dict(trace=[[e[0], e[1]] for e in trace], acceptance_rate=acc,
                                        oracle_matching_prefix=same, events=len(trace)))
            print(f"[e2e:{case['name']}] call {call}: acceptance {acc:.4f}, events {len(trace)}, "
                  f"oracle matches first {same} events ({time.time() - t0:.1f}s)")
        # autoregressive baseline trace (decoding.py:14-37)
        trace = []
        with rh.traced_random(CounterNoise(case["noise_seed"]), trace):
            ref.decoding.Autoregressive(tok, ge, ids, max_len=case["ar_len"], top_k=-1, top_p=top_p, temperature=T)
        eng.kv_cache.reset()
        otoks = orc.autoregressive(eng, ids.numpy(), case["ar_len"], CounterNoise(case["noise_seed"]))
        rtoks = [e[1] for e in trace if e[0] == "sample"]
        record["autoregressive"] = dict(tokens=rtoks, oracle_equal=(rtoks == otoks))
        print(f"[e2e:{case['name']}] AR tokens equal to oracle: {rtoks == otoks}")
        with open(os.path.join(HERE, f"e2e_{case['name']}.json"), "w") as f:
            json.dump(record, f)


def make_tree():
    """Sequoia tree path: the reference's SpecTree (utils/SpecTree_TP.py) on the functional reference layers, see
    oracle/ref_tree_harness.py.  Stores every round's 512 tree tokens, accepted tokens and random draws."""
    from oracle import ref_tree_harness as th
    from triforce_b200.spectree import load_grow_map
    case = gi.TREE_CASE
    ts = named_config(case["target"])
    sd = numpy_state_dict(ts, case["target_seed"])
    P, B, c, T = case["prefill"], case["budget"], case["chunk"], case["tree_size"]
    eng = th.RefTreeEngine(ts, sd, P, 64, B, c, T)
    ref = th.load_tree_reference()
    gm = load_grow_map(str(T))
    calls, gather = th.build_sampling(gm, case["temperature"])
    noise = CounterNoise(case["noise_seed"])
    trace, rounds = [], []
    with th.traced_tree_random(noise, trace):
        st = ref.spectree.SpecTree(engine=eng, temperature=case["temperature"], top_p=case["top_p"], max_length=P + 64, grow_map=gm,
                                   residual_graph=th.get_residual, sampling_callables=calls, sample_gather_indices=gather,
                                   tokenizer=None, vocab_size=ts.vocab_size)
        ids = numpy_prompt(P, seed=case["prompt_seed"])[0]
        nt = st.prefill(prefix=ids)
        first = int(nt.reshape(-1)[0])
        for r in range(case["rounds"]):
            mark = len(trace)
            st.construct_grow_map(next_token=nt)
            tree_tokens = st.verify_tokens.tolist()
            seq_before = eng.kv_cache.seq_len
            nt, acc, toks = st.verify()
            rounds.append(dict(tree_tokens=tree_tokens, acc_count=int(acc), accept_tokens=[] if nt is None else [int(x) for x in toks.tolist()],
                               seq_len_before=int(seq_before), seq_len_after=int(eng.kv_cache.seq_len),
                               events=[[e[0], e[1]] for e in trace[mark:]]))
            print(f"[tree] round {r}: acc_count {acc}, accepted {rounds[-1]['accept_tokens']}")
            if nt is None:
                break
            nt = nt.unsqueeze(0)
    with open(os.path.join(HERE, "tree_512.json"), "w") as f:
        json.dump(dict(case=case, first_token=first, rounds=rounds), f)


def make_reference_files():
    """Fixtures of the reference's own files, for the CPU tests that compare with them:
      ref_dataset_gs.npz    `books`: 24 PG-19 books of the reference's data/pg19 (the first 12 rows of each file, text cut to 2000
                            characters); `lengths` / `ids`: the reference's get_dataset('gs') on them, as one jsonl file, with the
                            byte tokenizer of tests/test_dataset_cpu.py
      ref_tree_512.npz      the reference's tree/512.pt (lists as JSON, the mask bit-packed)
      ref_cli_flags.json    every add_argument flag of the reference's test/{on_chip,offloading_TP,offloading_seqouia}.py with its default
    """
    import importlib.util
    import re
    import shutil
    import tempfile

    books = []
    for name in ("pg19-test.json", "pg19-train.json"):
        with open(os.path.join(rh.REF_ROOT, "data", "pg19", name), encoding="utf-8") as f:
            rows = [json.loads(line) for line in f if line.strip()][:12]
        books += [{"text": r["text"][:2000]} for r in rows]

    from test_dataset_cpu import ByteTokenizer
    tmp = tempfile.mkdtemp()
    try:
        os.environ.update(HF_HOME=os.path.join(tmp, "hf"), HF_DATASETS_CACHE=os.path.join(tmp, "hf", "datasets"), HF_DATASETS_OFFLINE="1")
        os.makedirs(os.path.join(tmp, "data", "pg19"))
        with open(os.path.join(tmp, "data", "pg19", "sample.jsonl"), "w", encoding="utf-8") as f:
            for b in books:
                f.write(json.dumps(b) + "\n")
        spec = importlib.util.spec_from_file_location("ref_dataset", os.path.join(rh.REF_ROOT, "data", "dataset.py"))
        ref = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref)
        cwd = os.getcwd()
        os.chdir(tmp)  # the reference opens "data/pg19/" relative to the working directory
        try:
            gs = ref.get_dataset("gs", tokenizer=ByteTokenizer())
        finally:
            os.chdir(cwd)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(HERE, "ref_dataset_gs.npz"), books=np.array([b["text"] for b in books]), lengths=np.array([t.shape[-1] for t in gs], np.int64),
                        ids=np.concatenate([t.reshape(-1).numpy() for t in gs]).astype(np.int32))
    print(f"[reference files] get_dataset('gs'): {len(gs)} prompts")

    g = torch.load(os.path.join(rh.REF_ROOT, "tree", "512.pt"), weights_only=False)
    lists = {k: g[k] for k in ("roots", "branches", "Successors", "size")}
    np.savez_compressed(os.path.join(HERE, "ref_tree_512.npz"), lists=np.array(json.dumps(lists)),
                        mask=np.packbits(g["mask"].numpy() != 0, axis=1), depth=g["depth"].numpy())

    flags = {}
    for entry in ("on_chip", "offloading_TP", "offloading_seqouia"):
        with open(os.path.join(rh.REF_ROOT, "test", entry + ".py")) as f:
            src = f.read()
        flags[entry] = {}
        for flag, rest in re.findall(r"add_argument\('--(\w+)'(.*?)\)\n", src):
            m = re.search(r"default=([^,)]+)", rest)
            flags[entry][flag] = (m.group(1).strip().strip("'").strip('"') if m else
                                  "store_true" if "store_true" in rest else None)
    with open(os.path.join(HERE, "ref_cli_flags.json"), "w") as f:
        json.dump(flags, f, indent=1)


if __name__ == "__main__":
    which = sys.argv[1:] or ["retrieval", "sampling", "forward", "yarn_7b", "e2e", "tree", "reference_files"]
    with torch.inference_mode():
        if "retrieval" in which:
            make_retrieval_build()
        if "sampling" in which:
            make_sampling()
        if "forward" in which:
            make_forward()
        if "yarn_7b" in which:
            make_yarn_7b()
        if "e2e" in which:
            make_e2e()
        if "tree" in which:
            make_tree()
        if "reference_files" in which:
            make_reference_files()
