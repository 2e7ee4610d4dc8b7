#!/usr/bin/env python
"""Cross-encoder reranking throughput (CrossEncoderReranker) beside the reference-equivalent in the same run.

Workload: the pipeline's fine-ranking step -- Q queries x k = 192 coarse candidates (f_topk_2), top_n = 6 (r_topk),
max_length 512; passages U[64, 480] tokens, queries U[8, 48], seeded; XLM-R-large (24 L / 1024 d / 16 H / ffn 4096,
vocab 250002, 514 positions) and XLM-R-base (12 L / 768 d / 12 H / ffn 3072) shapes with random bf16-representable
weights (no checkpoints offline; speed does not depend on the values).

Reported per (model, Q): pairs/s, encoder TFLOP/s (BertEncoder.flops over the pairs' lengths / encoder stage time),
stage times (pack / encoder / head + order) from CUDA events, and the card name and power limit read in this run.
The reference-equivalent is what CrossEncoder.predict runs: the transformers fp32 model on the same GPU over
right-padded batches of 32, plus the sigmoid (tokenisation excluded on both sides).  Parity: 64 pairs of query 0,
GPU logits vs that fp32 model, within 1.5x the bf16 evaluation's own distance from fp32 + 0.02.

    python scripts/bench_rerank.py --out DIR [--models large,base] [--queries 1,16,64] [--ref-max-queries 16]
"""
import argparse
import copy
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from easyrag_b200 import _lib                                                     # noqa: E402
from easyrag_b200.batched import TopK                                             # noqa: E402
from easyrag_b200.encoder import BertConfig                                       # noqa: E402
from easyrag_b200.rerank import CrossEncoderModel, CrossEncoderReranker, random_cross_encoder_state   # noqa: E402
from oracle import rerank as orr                                                  # noqa: E402

SHAPES = {"large": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096),
          "base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072)}
CLS, PAD, SEP = 0, 1, 2          # XLM-R <s> <pad> </s>
MAX_LENGTH = 512


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, power, clk = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:            # the device name still comes from torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})"}


def workload(rng, vocab, n_docs, nq, k):
    passages = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(64, 481, n_docs)]
    queries = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(8, 49, nq)]
    ids = np.stack([rng.choice(n_docs, k, replace=False) for _ in range(nq)]).astype(np.int32)
    return passages, queries, ids


def hf_predict(model, pairs, batch=32):
    """CrossEncoder.predict's model part: right-padded batches, fp32 logits -> sigmoid."""
    out = []
    for b0 in range(0, len(pairs), batch):
        chunk = pairs[b0:b0 + batch]
        w = max(len(p) for p in chunk)
        ids = torch.full((len(chunk), w), PAD, dtype=torch.long)
        mask = torch.zeros(len(chunk), w, dtype=torch.long)
        for i, p in enumerate(chunk):
            ids[i, :len(p)] = torch.tensor(p)
            mask[i, :len(p)] = 1
        with torch.no_grad():
            lg = model(input_ids=ids.cuda(non_blocking=True), attention_mask=mask.cuda(non_blocking=True)).logits[:, 0]
        out.append(torch.sigmoid(lg.float()))
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--models", default="large,base")
    ap.add_argument("--queries", default="1,16,64")
    ap.add_argument("--k", type=int, default=192)
    ap.add_argument("--top-n", type=int, default=6)
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-max-queries", type=int, default=16, help="time the fp32 reference up to this many queries")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rerank: no CUDA device (this benchmark measures the GPU path only)")
    _lib.require_cuda()
    from transformers import XLMRobertaConfig, XLMRobertaForSequenceClassification
    out_dir = Path(a.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    info = card()
    results = []
    for name in a.models.split(","):
        sh = SHAPES[name]
        cfg = BertConfig(vocab_size=250002, max_position_embeddings=514, layer_norm_eps=1e-5, **sh)
        state = random_cross_encoder_state("roberta", cfg, a.seed)
        model = CrossEncoderModel("roberta", cfg, state, CLS, SEP, PAD, device="cuda")
        hf = XLMRobertaForSequenceClassification(XLMRobertaConfig(
            vocab_size=cfg.vocab_size, max_position_embeddings=514, type_vocab_size=1, pad_token_id=PAD,
            layer_norm_eps=1e-5, num_labels=1, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
            attn_implementation="eager", **sh))
        hf.load_state_dict(state, strict=False)
        hf = hf.eval().cuda()
        del state
        rng = np.random.default_rng(a.seed)
        for nq in [int(x) for x in a.queries.split(",")]:
            passages, queries, ids = workload(rng, cfg.vocab_size, a.docs, nq, a.k)
            rr = CrossEncoderReranker(model, passages, max_length=MAX_LENGTH)
            cand = TopK(torch.zeros(nq, a.k, device="cuda"), torch.from_numpy(ids).cuda(),
                        torch.full((nq,), a.k, dtype=torch.int32, device="cuda"))
            q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32).cuda()
            q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32).cuda()
            lens = np.diff(rr.pack(cand.ids, cand.counts, q_ptr, q_tok).cu_h)
            flops = model.flops(lens.tolist())
            rr.rerank(cand, q_ptr, q_tok, a.top_n)                                   # warm-up
            torch.cuda.synchronize()
            stages, walls = [], []
            for _ in range(a.reps):
                ev = []
                t0 = time.perf_counter()
                _, all_scores = rr.rerank(cand, q_ptr, q_tok, a.top_n, events=ev)
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
                stages.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
            st = np.median(np.array(stages), axis=0)
            wall = float(np.median(walls))
            rec = {"model": f"xlm-roberta-{name}", "queries": nq, "k": a.k, "top_n": a.top_n, "pairs": int(lens.size),
                   "tokens": int(lens.sum()), "wall_s": wall, "pairs_per_s": lens.size / wall,
                   "stage_ms": {"pack": float(st[0]), "encoder": float(st[1]), "head_order": float(st[2])},
                   "encoder_tflops": flops / (st[1] * 1e-3) / 1e12, "reps": a.reps, "card": info}
            # parity: 64 pairs of query 0 against the fp32 model, with the bf16 model as the noise floor
            if nq == [int(x) for x in a.queries.split(",")][0]:
                pairs = [orr.cross_encoder_inputs(queries[0], passages[int(d)], MAX_LENGTH, "roberta", CLS, SEP, PAD)[0]
                         for d in ids[0, :64]]
                ref = hf_predict(hf, pairs).double().cpu().numpy()
                hf16 = copy.deepcopy(hf).to(torch.bfloat16)
                ref16 = hf_predict(hf16, pairs).double().cpu().numpy()
                del hf16
                got = all_scores[0, :64].double().cpu().numpy()
                lg = lambda s: np.log(s) - np.log1p(-s)
                err, floor = float(np.abs(lg(got) - lg(ref)).max()), float(np.abs(lg(ref16) - lg(ref)).max())
                rec["parity"] = {"pairs": 64, "max_logit_err": err, "bf16_floor": floor,
                                 "max_score_err": float(np.abs(got - ref).max()),
                                 "pass": bool(err <= 1.5 * floor + 0.02)}
            if nq <= a.ref_max_queries:
                pairs = [orr.cross_encoder_inputs(queries[q], passages[int(d)], MAX_LENGTH, "roberta", CLS, SEP, PAD)[0]
                         for q in range(nq) for d in ids[q]]
                hf_predict(hf, pairs[:32])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                hf_predict(hf, pairs)
                torch.cuda.synchronize()
                ref_s = time.perf_counter() - t0
                rec["reference_fp32"] = {"wall_s": ref_s, "pairs_per_s": len(pairs) / ref_s,
                                         "speedup": ref_s / wall}
            else:
                rec["reference_fp32"] = "not measured at this size"
            print(json.dumps(rec), flush=True)
            results.append(rec)
            del rr
            torch.cuda.empty_cache()
        del model, hf
        torch.cuda.empty_cache()
    (out_dir / "bench_rerank.json").write_text(json.dumps(results, indent=1))
    bad = [r for r in results if "parity" in r and not r["parity"]["pass"]]
    if bad:
        sys.exit(f"bench_rerank: parity failed: {[r['parity'] for r in bad]}")


if __name__ == "__main__":
    main()
