#!/usr/bin/env python
"""Encoder-side measurement for BASELINE.json configs[1]: "GTE-base 768-d encode + cosine top-10, 100k chunks,
1k queries" on one H100 (SURVEY.md 8(d): tensor-bound; report TFLOP/s vs the measured bf16 peak).

    python bench_encode.py [--arch bert|qwen2] [--chunks N] [--batch 512]         # one JSON line
    python bench.py --workload encode                                              # the same block as the bench line
    python bench.py                                                                # default line carries it as "encode"

Reference call sites: GTEEmbedding._embed (gte_embeddings.py:59-72), HuggingFaceEmbedding._embed
(hf_embeddings.py:118-123), the ingestion loop that embeds every chunk (pipeline.py:100-118,141-158).
Random-init weights of the named architecture (no checkpoints offline), synthetic token ids, chunk length
U[64,512], query length U[8,48].  The corpus rows are written by the pooling kernel straight into the dense index
matrix (no Python lists); queries are encoded and searched against that matrix.  Chunks shard across ranks
(plain data parallel, no collective on the data path).
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

SEED = 20240922 + 2


def build_model(arch: str, layers: int, d: int, dev):
    from easyrag_b200.encoder import BertConfig, BertEncoder, Qwen2Config, Qwen2Encoder, random_state
    if arch == "bert":
        cfg = BertConfig(vocab_size=21128, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                         num_attention_heads=d // 64, max_position_embeddings=512)
        state = random_state("bert", cfg, 1)
        return cfg, state, BertEncoder(cfg, state, device=dev)
    cfg = Qwen2Config(vocab_size=151646, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                      num_attention_heads=d // 64, num_key_value_heads=max(1, d // 64 // 3),
                      max_position_embeddings=1024)
    state = random_state("qwen2", cfg, 1)
    return cfg, state, Qwen2Encoder(cfg, state, device=dev)


def make_batches(lens: torch.Tensor, batch: int, vocab: int, dev, seed: int):
    """Packed batches built with tensor ops only (100k sequences): ids, cu_seqlens, positions on the device."""
    from easyrag_b200.encoder import PackedBatch
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    out = []
    for i in range(0, lens.numel(), batch):
        part = lens[i:i + batch].to(dev)
        cu = torch.zeros(part.numel() + 1, dtype=torch.int64, device=dev)
        torch.cumsum(part, 0, out=cu[1:])
        total = int(cu[-1])
        ids = torch.randint(1, vocab, (total,), generator=g, device=dev, dtype=torch.int32)
        pos = (torch.arange(total, device=dev) - torch.repeat_interleave(cu[:-1], part)).to(torch.int32)
        mx = int(part.max())
        out.append(PackedBatch(ids=ids, cu=cu.to(torch.int32), positions=pos, max_len=mx, n_seq=part.numel(), max_pos=mx))
    return out


def encode_block(dev, arch: str = "bert", chunks: int = 100_000, queries: int = 1_000, batch: int = 512, layers: int = 12,
                 dim: int = 768, steps: int = 3, rank: int = 0, world: int = 1, parity_seqs: int = 6,
                 len_min: int = 64, len_max: int = 512) -> dict:
    """The measured block; every rank calls it, every rank returns the same dict (times are the max over ranks)."""
    import torch.distributed as dist
    from easyrag_b200 import _lib, batched
    from easyrag_b200.index import DenseIndex
    from easyrag_b200.dist import shard_bounds
    _lib.require_cuda()
    L = _lib.lib()
    cfg, state, model = build_model(arch, layers, dim, dev)
    g = torch.Generator().manual_seed(SEED)
    lens_all = torch.randint(len_min, len_max + 1, (chunks,), generator=g)
    qlens = torch.randint(8, 49, (queries,), generator=g)
    lo, hi = shard_bounds(chunks, world, rank)
    lens = lens_all[lo:hi]
    cb = make_batches(lens, batch, cfg.vocab_size, dev, SEED + 1 + rank)
    qb = make_batches(qlens, batch, cfg.vocab_size, dev, SEED + 1000)
    index = DenseIndex(None, device=dev, dim=dim, capacity=int(lens.numel()), row_lo=lo)

    def encode_corpus():
        index.n_rows = 0
        for b in cb:
            model.embed_packed(b, out_bf16=index.rows_for_append(b.n_seq))     # pooled rows land in the corpus matrix
            index.commit(b.n_seq)

    def encode_queries(out):
        o = 0
        for b in qb:
            model.embed_packed(b, out_bf16=out[o:o + b.n_seq])
            o += b.n_seq

    def timed(fn):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms = torch.tensor([a.elapsed_time(b)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    for b in cb[:3]:                                      # warm-up: 3 batches
        model.embed_packed(b)
    torch.cuda.synchronize()
    _lib.check(L.ezr_profile_reset())
    _lib.check(L.ezr_profile_enable(1))
    launches0 = L.ezr_launch_count()
    ms_corpus = timed(encode_corpus)
    launches = L.ezr_launch_count() - launches0
    _lib.check(L.ezr_profile_enable(0))
    prof = {n: _lib.profile_read(n) for n in ("enc_gemm", "enc_attn", "enc_other")}
    attn_kernel = L.ezr_attn_last_kernel().decode()
    flops_local = model.flops(lens.tolist())
    attn_flops_local = float(sum(cfg.num_hidden_layers * 4 * n * n * dim for n in lens.tolist()))
    # queries: encode + cosine top-10 against the corpus rows just produced (this rank's shard)
    qv = torch.empty(queries, dim, dtype=torch.bfloat16, device=dev)
    encode_queries(qv)
    torch.cuda.synchronize()

    def query_steps():
        for _ in range(steps):
            encode_queries(qv)
            batched.dense_topk(index, qv, 10)
    ms_query = timed(query_steps) / steps
    peaks = {}
    pk = ROOT / "MEASURED_PEAKS.json"
    if pk.exists():
        peaks = json.loads(pk.read_text())
    long_run = ms_corpus > 2000.0
    key = "bf16_tflops_sustained" if long_run else "bf16_tflops"
    peak = float(peaks.get(key, 989.0))                  # H100 SXM data sheet, dense bf16
    gemm_ms, attn_ms = prof["enc_gemm"][0], prof["enc_attn"][0]
    gemm_tf = (flops_local - attn_flops_local) / (gemm_ms * 1e-3) / 1e12 if gemm_ms else None
    attn_tf = attn_flops_local / (attn_ms * 1e-3) / 1e12 if attn_ms else None
    # parity of a few sequences against the fp32 oracle on the same bf16-rounded weights (north star: cosine 1e-3)
    parity = None
    if parity_seqs > 0 and rank == 0:
        parity = oracle_parity(arch, cfg, state, model, cb[0], parity_seqs)
    tokens_all = int(lens_all.sum())
    return {
        "arch": arch, "layers": layers, "dim": dim, "chunks": chunks, "tokens": tokens_all, "batch_sequences": batch,
        "chunk_len": f"U[{len_min},{len_max}]", "query_len": "U[8,48]", "n_gpus": world,
        "encode_s": ms_corpus * 1e-3, "chunks_per_s": chunks / (ms_corpus * 1e-3),
        "tokens_per_s": tokens_all / (ms_corpus * 1e-3),
        "model_tflops_per_gpu": flops_local / (ms_corpus * 1e-3) / 1e12,
        "gemm": {"ms": gemm_ms, "launches": prof["enc_gemm"][1], "tflops": gemm_tf,
                 "frac_of_measured_bf16": gemm_tf / peak if gemm_tf else None},
        "attention": {"kernel": attn_kernel, "ms": attn_ms, "launches": prof["enc_attn"][1], "tflops": attn_tf,
                      "frac_of_measured_bf16": attn_tf / peak if attn_tf else None},
        "other_ms": prof["enc_other"][0], "gpu_launches": int(launches),
        "queries": {"n": queries, "encode_plus_top10_ms": ms_query, "queries_per_s": queries / (ms_query * 1e-3),
                    "corpus_rows_searched": index.n_rows},
        "peak_tflops": peak, "peak_source": f"MEASURED_PEAKS.json {key}" if key in peaks else "H100 SXM data sheet",
        "timing": "CUDA events around the whole corpus encode (max over ranks); per-kernel sums from ezr_profile_* events",
        "corpus_rows_written_in_place": True, "dtype": "bf16", "data": "synthetic ids, random-init weights",
        "parity": parity,
    }


def oracle_parity(arch, cfg, state, model, batch, n_seq: int) -> dict:
    """First ``n_seq`` sequences of a batch through the fp32 CPU oracle (oracle/encoder.py) and through the kernels:
    largest difference between the two cosine-score matrices of those sequences."""
    from oracle import encoder as oenc
    from easyrag_b200.encoder import PackedBatch
    cu = batch.cu[:n_seq + 1].cpu()
    total = int(cu[-1])
    sub = PackedBatch(ids=batch.ids[:total], cu=batch.cu[:n_seq + 1].contiguous(), positions=batch.positions[:total],
                      max_len=int((cu[1:] - cu[:-1]).max()), n_seq=n_seq)
    got = model.embed_packed(sub)[1].cpu()
    ids = batch.ids[:total].cpu().tolist()
    seqs = [ids[int(cu[i]):int(cu[i + 1])] for i in range(n_seq)]
    import torch.nn.functional as F
    if arch == "bert":
        ref = oenc.bert_embed(state, cfg, seqs, pooling="cls")
        ref_bf16 = oenc.bert_embed(state, cfg, seqs, pooling="cls", dtype=torch.bfloat16)
    else:
        iid, mask = oenc.pad_left(seqs)
        ref = oenc.gte_embed(state, cfg, iid, mask)
        ref_bf16 = oenc.gte_embed(state, cfg, iid, mask, torch.bfloat16)
    ref_bf16 = F.normalize(ref_bf16.float(), dim=1)
    got = F.normalize(got, dim=1)
    # the bar of tests/test_gpu_encoder.py: every embedding within 1e-3 (cosine) of the fp32 oracle's, and the pairwise
    # cosine scores (what a retriever sees) within 1e-3 of the fp32 scores beyond the floor ANY bf16 evaluation of
    # these weights has (the oracle itself run in bf16 on the CPU)
    self_cos = float((got * ref).sum(1).min())
    err = float(((got @ got.T) - (ref @ ref.T)).abs().max())
    floor = float(((ref_bf16 @ ref_bf16.T) - (ref @ ref.T)).abs().max())
    return {"sequences": n_seq, "min_cosine_to_fp32_oracle": self_cos, "pairwise_cosine_max_abs_err": err,
            "bf16_oracle_floor": floor, "tol": 1e-3, "ok": bool(self_cos >= 1 - 1e-3 and err <= floor + 1e-3)}


def main(from_bench=None):
    import os
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="bert", choices=["bert", "qwen2"])
    ap.add_argument("--chunks", type=int, default=100_000)
    ap.add_argument("--enc-queries", type=int, default=1_000)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--enc-dim", type=int, default=768)
    ap.add_argument("--enc-steps", type=int, default=3)
    ap.add_argument("--len-min", type=int, default=64)
    ap.add_argument("--len-max", type=int, default=512)
    args = ap.parse_known_args()[0]
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    blk = encode_block(dev, args.arch, args.chunks, args.enc_queries, args.batch, args.layers, args.enc_dim,
                       args.enc_steps, rank, world, len_min=args.len_min, len_max=args.len_max)
    if rank == 0:
        if from_bench is not None:
            line = {"metric": "chunks/sec GTE-base-shaped 768-d encode (configs[1])", "value": blk["chunks_per_s"],
                    "unit": "chunks/s", "n_gpus": world, "steps": 1, "warmup": 3, "ms_per_step": blk["encode_s"] * 1e3,
                    "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "bf16",
                    "data": "synthetic", "config": {"workload": "configs[1]: GTE-base 768-d encode + cosine top-10, "
                                                                f"{args.chunks} chunks, {args.enc_queries} queries"},
                    "gpu_launches": blk["gpu_launches"], "encode": blk}
        else:
            line = dict(bench="encode", **blk)
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
