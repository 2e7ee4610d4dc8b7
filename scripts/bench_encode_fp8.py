#!/usr/bin/env python
"""FP8 (e4m3) against bf16 encoder GEMMs on one GPU, in the same run.

    python scripts/bench_encode_fp8.py --out DIR [--m 147456] [--chunks 20000] [--qwen-chunks 1000]

Writes DIR/bench_encode_fp8.json and prints it.  Three blocks:
  gemm     per-GEMM kernel time (CUDA events over --reps launches, median of 3 alternating bf16 / fp8 rounds) and
           TFLOP/s = 2 M N K / time, at the gte-Qwen2-7B, BERT-base and BERT-large layer shapes, M tokens; the fp8
           time excludes quantising the activations, reported separately as quant_ms (per-row quantiser on the
           GEMM's input, which the encoders run before o_proj / down_proj and fuse into the norms elsewhere).
  encode   chunks/s of the bench_encode.py workload (12 layers, d 768, chunks of U[64,512] tokens) and of a 28-layer
           Qwen2 at d 3584 (FFN 18944) on fewer chunks, bf16 and fp8, one timed pass each after a warm-up.
  overlap  the overlap of dense top-10 lists between the corpus encoded in bf16 and in fp8 (random weights: a
           measure of how far the two encodings move the ranking, not of retrieval quality).
GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

# (name, K, N, epilogue): the layer GEMMs; gate/up is one GEMM of N = 2 ffn with the SwiGLU epilogue
SHAPES = [
    ("qwen2-7b qkv", 3584, 4608, 0), ("qwen2-7b o", 3584, 3584, 0), ("qwen2-7b gate/up", 3584, 2 * 18944, 2),
    ("qwen2-7b down", 18944, 3584, 0),
    ("bert-base qkv", 768, 2304, 0), ("bert-base o", 768, 768, 0), ("bert-base ffn1", 768, 3072, 1),
    ("bert-base ffn2", 3072, 768, 0),
    ("bert-large qkv", 1024, 3072, 0), ("bert-large o", 1024, 1024, 0), ("bert-large ffn1", 1024, 4096, 1),
    ("bert-large ffn2", 4096, 1024, 0),
]


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"nvidia_smi": r.stdout.strip(), "torch_name": torch.cuda.get_device_name()}


def _event_ms(fn, reps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def gemm_block(m: int, reps: int) -> list:
    from easyrag_b200 import encoder as enc
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(7)
    rows = []
    for name, k, n, epi in SHAPES:
        a = torch.randn(m, k, generator=g, device=dev).to(torch.bfloat16)
        w = (torch.randn(n, k, generator=g, device=dev) * 0.02).to(torch.bfloat16)
        a8, sa = enc.quant_rows(a)
        w8, sw = enc.quant_weight(w)
        n_out = n // 2 if epi == 2 else n
        out = torch.empty(m, n_out, dtype=torch.bfloat16, device=dev)
        f_bf16 = lambda: enc.gemm(a, w, out=out, epilogue=epi)
        f_fp8 = lambda: enc.gemm_fp8(a8, sa, w8, sw, out=out, epilogue=epi)
        f_q = lambda: enc.quant_rows(a, a8, sa)
        for f in (f_bf16, f_fp8, f_q):                          # warm-up
            f()
        torch.cuda.synchronize()
        t = {"bf16": [], "fp8": [], "quant": []}
        for _ in range(3):                                      # alternate the two kernels
            t["bf16"].append(_event_ms(f_bf16, reps))
            t["fp8"].append(_event_ms(f_fp8, reps))
            t["quant"].append(_event_ms(f_q, reps))
        med = {kk: sorted(v)[1] for kk, v in t.items()}
        flop = 2.0 * m * n * k
        rows.append({"gemm": name, "M": m, "K": k, "N": n, "epilogue": ["none", "gelu", "swiglu"][epi],
                     "bf16_ms": med["bf16"], "fp8_ms": med["fp8"], "quant_ms": med["quant"],
                     "bf16_tflops": flop / med["bf16"] / 1e9, "fp8_tflops": flop / med["fp8"] / 1e9,
                     "speedup": med["bf16"] / med["fp8"],
                     "fp8_tflops_incl_quant": flop / (med["fp8"] + med["quant"]) / 1e9,
                     "timing": f"CUDA events over {reps} launches, median of 3 alternating rounds"})
        print(json.dumps(rows[-1]), flush=True)
        del a, w, a8, w8, out
        torch.cuda.empty_cache()
    return rows


def encode_block(arch: str, layers: int, d: int, ffn: int, chunks: int, batch: int) -> dict:
    import bench_encode as be
    from easyrag_b200 import batched
    from easyrag_b200.encoder import BertConfig, BertEncoder, Qwen2Config, Qwen2Encoder, random_state
    from easyrag_b200.index import DenseIndex
    dev = "cuda"
    if arch == "bert":
        cfg = BertConfig(vocab_size=21128, hidden_size=d, intermediate_size=ffn, num_hidden_layers=layers,
                         num_attention_heads=d // 64, max_position_embeddings=512)
        state = random_state("bert", cfg, 1)
        make = lambda p: BertEncoder(cfg, state, device=dev, precision=p)
    else:
        cfg = Qwen2Config(vocab_size=32000, hidden_size=d, intermediate_size=ffn, num_hidden_layers=layers,
                          num_attention_heads=d // 128, num_key_value_heads=4, max_position_embeddings=1024,
                          rope_theta=1e6)
        # one layer of random weights shared by every layer: the host copy of 28 distinct 7B-width layers would
        # need ~26 GB; speed does not depend on the values
        one = random_state("qwen2", Qwen2Config(**{**cfg.__dict__, "num_hidden_layers": 1}), 1)
        state = {k: v for k, v in one.items() if not k.startswith("layers.")}
        for i in range(layers):
            state.update({k.replace("layers.0.", f"layers.{i}."): v for k, v in one.items() if k.startswith("layers.0.")})
        make = lambda p: Qwen2Encoder(cfg, state, device=dev, precision=p)
    g = torch.Generator().manual_seed(be.SEED)
    lens = torch.randint(64, 513, (chunks,), generator=g)
    cb = be.make_batches(lens, batch, cfg.vocab_size, dev, be.SEED + 1)
    qb = be.make_batches(torch.randint(8, 49, (1000,), generator=g), batch, cfg.vocab_size, dev, be.SEED + 1000)
    res = {"arch": arch, "layers": layers, "dim": d, "ffn": ffn, "chunks": chunks, "tokens": int(lens.sum()),
           "chunk_len": "U[64,512]", "batch_sequences": batch}
    tops = {}
    for prec in ("bf16", "fp8"):
        model = make(prec)
        index = DenseIndex(None, device=dev, dim=d, capacity=chunks)
        for b in cb[:2]:
            model.embed_packed(b)
        torch.cuda.synchronize()

        def encode():
            index.n_rows = 0
            for b in cb:
                model.embed_packed(b, out_bf16=index.rows_for_append(b.n_seq))
                index.commit(b.n_seq)
        ms = _event_ms(encode, 1)
        qv = torch.empty(1000, d, dtype=torch.bfloat16, device=dev)
        o = 0
        for b in qb:
            model.embed_packed(b, out_bf16=qv[o:o + b.n_seq])
            o += b.n_seq
        tops[prec] = batched.dense_topk(index, qv, 10).ids.cpu()
        res[prec] = {"encode_s": ms * 1e-3, "chunks_per_s": chunks / (ms * 1e-3),
                     "model_tflops": model.flops(lens.tolist()) / (ms * 1e-3) / 1e12, "timing": "single run"}
        del model, index
        torch.cuda.empty_cache()
    a, b = tops["bf16"], tops["fp8"]
    overlap = sum(len(set(a[i].tolist()) & set(b[i].tolist())) for i in range(a.shape[0])) / a.numel()
    res["speedup"] = res["fp8"]["chunks_per_s"] / res["bf16"]["chunks_per_s"]
    res["top10_overlap_bf16_vs_fp8"] = overlap
    res["overlap_note"] = "random-weight model, queries encoded with the same precision: not a retrieval-quality figure"
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--m", type=int, default=147456)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--chunks", type=int, default=20000)
    ap.add_argument("--qwen-chunks", type=int, default=1000)
    ap.add_argument("--skip-encode", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode_fp8 needs a CUDA device")
    from easyrag_b200 import _lib
    _lib.require_cuda()
    out = {"gpu": gpu_info(), "gemm": gemm_block(args.m, args.reps)}
    if not args.skip_encode:
        out["encode"] = [encode_block("bert", 12, 768, 3072, args.chunks, 512),
                         encode_block("qwen2", 28, 3584, 18944, args.qwen_chunks, 64)]
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "bench_encode_fp8.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
