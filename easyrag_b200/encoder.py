"""Chunk / query embedding forward pass on the GPU: Qwen2-shaped (GTE) and BERT-shaped (BGE / GTE-base) encoders.

Replaces the model call inside ``GTEEmbedding._embed`` (gte_embeddings.py:59-72 -> the vendored
``Qwen2Model.forward`` run bidirectionally, modeling_qwen.py:956-1116) and inside
``HuggingFaceEmbedding._embed`` (hf_embeddings.py:112-123 -> SentenceTransformer.encode on a BERT
encoder).  The host code is Python, as in the reference; every arithmetic step is a CUDA kernel behind
the C ABI (csrc/encoder/*.cu): wgmma GEMMs with fused bias / GELU / SwiGLU / residual epilogues,
tensor-core bidirectional attention over packed sequences, RMSNorm / LayerNorm / RoPE / pooling kernels.
torch tensors are only the device buffers.

Sequences are packed (no padding tokens): the reference pads every batch to its longest text and
masks (gte_embeddings.py:63); packing computes exactly the same per-token function for real tokens
and skips the rest.  ``pos_offset`` reproduces the one observable side effect of left padding in the
reference: position ids are column indices (modeling_qwen.py:1003-1008), so a sequence of length n in
a batch of width L starts at position L - n.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib

EPI_NONE, EPI_GELU, EPI_SWIGLU = 0, 1, 2
POOL_LAST, POOL_CLS, POOL_MEAN = 0, 1, 2


# ------------------------------------------------------------------------------- thin op wrappers
def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, epilogue: int = EPI_NONE) -> torch.Tensor:
    """out = epi(a @ w.T + bias) (+ residual);  a [M,K], w [N,K] bf16 row-major."""
    L = _lib.lib()
    m, k = a.shape
    n = w.shape[0]
    n_out = n // 2 if epilogue == EPI_SWIGLU else n
    if out is None:
        out = torch.empty(m, n_out, dtype=torch.bfloat16, device=a.device)
    _lib.check(L.ezr_gemm_bf16(_lib.ptr(a), m, k, a.stride(0), _lib.ptr(w), n, w.stride(0), _lib.ptr(bias),
                               _lib.ptr(residual), residual.stride(0) if residual is not None else 0, _lib.ptr(out),
                               out.stride(0), epilogue, _lib.stream_ptr()), "ezr_gemm_bf16")
    return out


def attention(qkv: torch.Tensor, cu: torch.Tensor, max_len: int, n_heads: int, n_kv: int, head_dim: int,
              out: Optional[torch.Tensor] = None, causal: bool = False) -> torch.Tensor:
    """Attention over packed q|k|v rows; ``causal=True``: row r of a sequence sees its keys 0..r (ezr_attn_causal)."""
    L = _lib.lib()
    t = qkv.shape[0]
    if out is None:
        out = torch.empty(t, n_heads * head_dim, dtype=torch.bfloat16, device=qkv.device)
    name = "ezr_attn_causal" if causal else "ezr_attn_bidir"
    _lib.check(getattr(L, name)(_lib.ptr(qkv), t, qkv.stride(0), _lib.ptr(cu), cu.numel() - 1, max_len, n_heads, n_kv,
                                head_dim, 1.0 / math.sqrt(head_dim), _lib.ptr(out), out.stride(0), _lib.stream_ptr()),
               name)
    return out


def rmsnorm(x: torch.Tensor, gamma: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    L = _lib.lib()
    if out is None:
        out = torch.empty_like(x)
    _lib.check(L.ezr_rmsnorm(_lib.ptr(x), x.stride(0), _lib.ptr(gamma), eps, x.shape[0], x.shape[1], _lib.ptr(out),
                             out.stride(0), _lib.stream_ptr()), "ezr_rmsnorm")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    L = _lib.lib()
    if out is None:
        out = torch.empty_like(x)
    _lib.check(L.ezr_layernorm(_lib.ptr(x), x.stride(0), _lib.ptr(gamma), _lib.ptr(beta), eps, x.shape[0], x.shape[1],
                               _lib.ptr(out), out.stride(0), _lib.stream_ptr()), "ezr_layernorm")
    return out


def gemm_fp8(a8: torch.Tensor, sa: torch.Tensor, w8: torch.Tensor, sw: torch.Tensor, bias: Optional[torch.Tensor] = None,
             residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
             epilogue: int = EPI_NONE) -> torch.Tensor:
    """out = epi(diag(sa) a8 @ w8.T diag(sw) + bias) (+ residual);  a8 [M,K], w8 [N,K] float8_e4m3fn, sa [M] / sw [N]
    float32 power-of-two scales (quant_rows / quant_weight).  SwiGLU weights interleave gate / up rows per 64
    (``_interleave_gate_up(.., block=64)``)."""
    L = _lib.lib()
    m, k = a8.shape
    n = w8.shape[0]
    n_out = n // 2 if epilogue == EPI_SWIGLU else n
    if out is None:
        out = torch.empty(m, n_out, dtype=torch.bfloat16, device=a8.device)
    _lib.check(L.ezr_gemm_fp8(_lib.ptr(a8), _lib.ptr(sa), m, k, a8.stride(0), _lib.ptr(w8), _lib.ptr(sw), n, w8.stride(0),
                              _lib.ptr(bias), _lib.ptr(residual), residual.stride(0) if residual is not None else 0,
                              _lib.ptr(out), out.stride(0), epilogue, _lib.stream_ptr()), "ezr_gemm_fp8")
    return out


def _fp8_dest(x: torch.Tensor, out8: Optional[torch.Tensor], scale: Optional[torch.Tensor]):
    if out8 is None:
        out8 = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    if scale is None:
        scale = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    return out8, scale


def quant_rows(x: torch.Tensor, out8: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 [rows, cols] -> (e4m3 [rows, cols], float32 [rows]): one power-of-two scale per row (ezr_quant_rows_fp8)."""
    L = _lib.lib()
    out8, scale = _fp8_dest(x, out8, scale)
    _lib.check(L.ezr_quant_rows_fp8(_lib.ptr(x), x.stride(0), x.shape[0], x.shape[1], _lib.ptr(out8), out8.stride(0),
                                    _lib.ptr(scale), _lib.stream_ptr()), "ezr_quant_rows_fp8")
    return out8, scale


def quant_weight(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """nn.Linear weight bf16 [n, k] -> (e4m3 [n, k], float32 [n]): one power-of-two scale per output channel."""
    L = _lib.lib()
    w8, scale = _fp8_dest(w, None, None)
    _lib.check(L.ezr_quant_weight_fp8(_lib.ptr(w), w.stride(0), w.shape[0], w.shape[1], _lib.ptr(w8), w8.stride(0),
                                      _lib.ptr(scale), _lib.stream_ptr()), "ezr_quant_weight_fp8")
    return w8, scale


def rmsnorm_fp8(x: torch.Tensor, gamma: torch.Tensor, eps: float, out8: Optional[torch.Tensor] = None,
                scale: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
    """rmsnorm's bf16 row (also stored to ``out`` when given), quantised per row -> (e4m3, float32 scales)."""
    L = _lib.lib()
    out8, scale = _fp8_dest(x, out8, scale)
    _lib.check(L.ezr_rmsnorm_fp8(_lib.ptr(x), x.stride(0), _lib.ptr(gamma), eps, x.shape[0], x.shape[1], _lib.ptr(out),
                                 out.stride(0) if out is not None else 0, _lib.ptr(out8), out8.stride(0), _lib.ptr(scale),
                                 _lib.stream_ptr()), "ezr_rmsnorm_fp8")
    return out8, scale


def layernorm_fp8(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
                  out8: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None):
    """layernorm's bf16 row (also stored to ``out`` when given), quantised per row -> (e4m3, float32 scales)."""
    L = _lib.lib()
    out8, scale = _fp8_dest(x, out8, scale)
    _lib.check(L.ezr_layernorm_fp8(_lib.ptr(x), x.stride(0), _lib.ptr(gamma), _lib.ptr(beta), eps, x.shape[0],
                                   x.shape[1], _lib.ptr(out), out.stride(0) if out is not None else 0, _lib.ptr(out8),
                                   out8.stride(0), _lib.ptr(scale), _lib.stream_ptr()), "ezr_layernorm_fp8")
    return out8, scale


# One layer loop per encoder serves both precisions.  A GEMM operand is a bf16 tensor, or an (e4m3, float32 scales)
# pair in fp8 mode; ``q`` is the pair of buffers an operand is quantised into, None in bf16 mode.
def _linear(a, w, **kw) -> torch.Tensor:
    """gemm, or gemm_fp8 for a weight ``_weight`` stored as (e4m3, scales)."""
    return gemm_fp8(*a, *w, **kw) if isinstance(w, tuple) else gemm(a, w, **kw)


def _operand(x: torch.Tensor, q):
    """bf16 ``x`` as a GEMM operand: itself, or quantised per row into ``q``."""
    return x if q is None else quant_rows(x, *q)


def _norm(x: torch.Tensor, gamma: torch.Tensor, beta: Optional[torch.Tensor], eps: float, out, q):
    """RMSNorm (``beta`` None) or LayerNorm of ``x`` as a GEMM operand: the bf16 row written to ``out``, or quantised
    into ``q`` by the same kernel, which then also writes the bf16 row to ``out`` unless it is None."""
    if q is None:
        return rmsnorm(x, gamma, eps, out=out) if beta is None else layernorm(x, gamma, beta, eps, out=out)
    return rmsnorm_fp8(x, gamma, eps, *q, out=out) if beta is None else layernorm_fp8(x, gamma, beta, eps, *q, out=out)


PRECISIONS = ("bf16", "fp8")


def _check_precision(precision: str) -> None:
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")


def _dest(out_bf16: Optional[torch.Tensor], n: int, d: int, device) -> torch.Tensor:
    if out_bf16 is None:
        return torch.empty(n, d, dtype=torch.bfloat16, device=device)
    if out_bf16.shape != (n, d) or out_bf16.dtype != torch.bfloat16 or not out_bf16.is_contiguous():
        raise ValueError("out_bf16 must be a contiguous bf16 [n_seq, dim] tensor (a row slice of the corpus matrix)")
    return out_bf16


def _pool(enc, batch: PackedBatch, out_bf16: Optional[torch.Tensor], pool: int, gamma: Optional[torch.Tensor],
          eps: float, l2: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``enc.hidden(batch)`` pooled per sequence, RMS-normed with ``gamma`` unless it is None, and L2-normalised in
    mode ``l2`` (ezr_pool_normalize) -> (bf16 [B, d], float32 copy)."""
    x = enc.hidden(batch)
    d = enc.cfg.hidden_size
    out_b = _dest(out_bf16, batch.n_seq, d, enc.device)
    out_f = torch.empty(batch.n_seq, d, dtype=torch.float32, device=enc.device)
    with torch.cuda.device(enc.device):
        _lib.check(_lib.lib().ezr_pool_normalize(_lib.ptr(x), x.stride(0), _lib.ptr(batch.cu), batch.n_seq, pool,
                                                 int(gamma is not None), _lib.ptr(gamma), eps, l2, d, _lib.ptr(out_b),
                                                 _lib.ptr(out_f), _lib.stream_ptr()), "ezr_pool_normalize")
    return out_b, out_f


# ------------------------------------------------------------------------------------- packing
@dataclass
class PackedBatch:
    ids: torch.Tensor          # int32 [T]
    cu: torch.Tensor           # int32 [B+1]
    positions: torch.Tensor    # int32 [T]
    max_len: int
    n_seq: int
    max_pos: Optional[int] = None   # largest position id + 1 (host-known when built by from_lists / from_padded)
    types: Optional[torch.Tensor] = None   # int32 [T] token type ids (BERT-shaped encoders); None = type 0 everywhere

    def check_positions(self, limit: int) -> None:
        """The rope / position-embedding kernels index tables of ``limit`` rows; an id past the table would read
        the clamped last row and give a silently wrong embedding, so it is an error here."""
        if self.max_pos is None:
            self.max_pos = int(self.positions.max()) + 1 if self.positions.numel() else 0
        if self.max_pos > limit:
            raise ValueError(f"position id {self.max_pos - 1} outside the model's table of {limit} positions "
                             f"(lower max_length or use a model with a longer max_position_embeddings)")

    @staticmethod
    def from_lists(seqs: Sequence[Sequence[int]], device, pos_offset: Optional[Sequence[int]] = None) -> "PackedBatch":
        lens = [len(s) for s in seqs]
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        flat = [int(t) for s in seqs for t in s]
        pos = []
        for i, n in enumerate(lens):
            o = int(pos_offset[i]) if pos_offset is not None else 0
            pos.extend(range(o, o + n))
        return PackedBatch(ids=torch.tensor(flat, dtype=torch.int32, device=device),
                           cu=torch.tensor(cu, dtype=torch.int32, device=device),
                           positions=torch.tensor(pos, dtype=torch.int32, device=device),
                           max_len=max(lens) if lens else 0, n_seq=len(lens), max_pos=(max(pos) + 1) if pos else 0)

    @staticmethod
    def from_padded(input_ids: torch.Tensor, attention_mask: torch.Tensor, device,
                    column_positions: bool = True) -> "PackedBatch":
        """HF tokenizer output ([B, L] ids + mask, left- or right-padded) -> packed.

        ``column_positions=True`` keeps the reference's position ids = column index (modeling_qwen.py:1003-1008).
        """
        ids = input_ids.to("cpu")
        mask = attention_mask.to("cpu").bool()
        b, l = ids.shape
        seqs, offs = [], []
        for i in range(b):
            cols = torch.nonzero(mask[i]).flatten()
            seqs.append(ids[i, cols].tolist())
            offs.append(int(cols[0]) if (column_positions and cols.numel()) else 0)
        return PackedBatch.from_lists(seqs, device, offs)


# ------------------------------------------------------------------------------------ Qwen2 (GTE)
@dataclass
class Qwen2Config:
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    num_key_value_heads: int
    max_position_embeddings: int = 8192
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1000000.0
    sliding_window: Optional[int] = None    # Qwen2's causal mask window (not implemented: longer causal inputs are refused)

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


def _bf16(t: torch.Tensor, device) -> torch.Tensor:
    return t.detach().to(device=device, dtype=torch.bfloat16).contiguous()


def _weight(t: torch.Tensor, device, precision: str):
    """A layer weight as the GEMMs of ``precision`` take it: bf16, or (e4m3, per-channel scales) with no bf16 copy kept."""
    w = _bf16(t, device)
    return w if precision == "bf16" else quant_weight(w)


def _interleave_gate_up(gate: torch.Tensor, up: torch.Tensor, block: int = 128) -> torch.Tensor:
    """[ffn, d] x2 -> [2*ffn, d] in blocks of ``block`` gate rows followed by the matching ``block`` up rows (SwiGLU
    epilogue: one GEMM tile holds both halves of the same outputs; 128 for the bf16 kernel's 256-column tiles, 64 for
    the fp8 kernel's 128-column tiles)."""
    ffn, d = gate.shape
    if ffn % 128:
        raise ValueError("intermediate_size must be a multiple of 128")
    g = gate.view(ffn // block, block, d)
    u = up.view(ffn // block, block, d)
    return torch.stack([g, u], dim=1).reshape(2 * ffn, d).contiguous()


class Qwen2Encoder:
    """Bidirectional Qwen2 stack + last-token pooling + L2 norm == GTEEmbedding._embed's model part.

    ``precision="fp8"`` holds the layer weights as e4m3 with per-channel scales only and runs every layer GEMM on
    the e4m3 kernel (activations quantised per row); embeddings, norms, attention, RoPE, pooling and the residual
    stream stay bf16.  Lossy: see DESIGN.md 4.5a for its error bound.

    ``causal=True`` runs the stack as ``Qwen2Model.forward(is_causal=True)`` does (modeling_qwen.py:1043-1051): every
    layer's attention lets token r of a sequence see tokens 0..r only; pooling stays last-token.  A sequence longer
    than ``cfg.sliding_window`` is refused: the window is not implemented."""

    def __init__(self, cfg: Qwen2Config, state: Dict[str, torch.Tensor], device="cuda", precision: str = "bf16",
                 causal: bool = False):
        _check_precision(precision)
        _lib.require_cuda()
        self.cfg = cfg
        self.precision = precision
        self.causal = bool(causal)
        self.device = torch.device(device)
        if cfg.head_dim not in (64, 128):
            raise ValueError("head_dim must be 64 or 128")
        dev = self.device
        g = lambda name: state[name]
        self.embed = _bf16(g("embed_tokens.weight"), dev)
        self.layers = []
        for i in range(cfg.num_hidden_layers):
            p = f"layers.{i}."
            wqkv = torch.cat([g(p + "self_attn.q_proj.weight"), g(p + "self_attn.k_proj.weight"),
                              g(p + "self_attn.v_proj.weight")], 0)
            bqkv = torch.cat([g(p + "self_attn.q_proj.bias"), g(p + "self_attn.k_proj.bias"),
                              g(p + "self_attn.v_proj.bias")], 0)
            block = 128 if precision == "bf16" else 64
            wgu = _interleave_gate_up(g(p + "mlp.gate_proj.weight").float(), g(p + "mlp.up_proj.weight").float(), block)
            self.layers.append(dict(
                ln1=_bf16(g(p + "input_layernorm.weight"), dev), wqkv=_weight(wqkv, dev, precision),
                bqkv=_bf16(bqkv, dev), wo=_weight(g(p + "self_attn.o_proj.weight"), dev, precision),
                ln2=_bf16(g(p + "post_attention_layernorm.weight"), dev), wgu=_weight(wgu, dev, precision),
                wdown=_weight(g(p + "mlp.down_proj.weight"), dev, precision)))
        self.norm = _bf16(g("norm.weight"), dev)
        # rotary tables exactly as Qwen2RotaryEmbedding builds them (modeling_qwen.py:100-133): fp32 math, cast to bf16
        hd = cfg.head_dim
        inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float().to(dev) / hd))
        t = torch.arange(cfg.max_position_embeddings, device=dev, dtype=torch.int64).type_as(inv_freq)
        freqs = torch.outer(t, inv_freq)
        self.cos = freqs.cos().to(torch.bfloat16).contiguous()
        self.sin = freqs.sin().to(torch.bfloat16).contiguous()

    @torch.no_grad()
    def hidden(self, batch: PackedBatch) -> torch.Tensor:
        """Last-layer hidden states BEFORE the final norm, [T, d] bf16."""
        L = _lib.lib()
        cfg = self.cfg
        t = batch.ids.numel()
        d, hd, H, KV = cfg.hidden_size, cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
        dev = self.device
        batch.check_positions(cfg.max_position_embeddings)
        if self.causal and cfg.sliding_window is not None and batch.max_len > cfg.sliding_window:
            raise ValueError(f"a sequence of {batch.max_len} tokens is longer than the causal sliding window of "
                             f"{cfg.sliding_window}, which this encoder does not implement")
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            x = torch.empty(t, d, dtype=torch.bfloat16, device=dev)
            _lib.check(L.ezr_embed_gather(_lib.ptr(batch.ids), t, _lib.ptr(self.embed), self.embed.stride(0),
                                          cfg.vocab_size, d, _lib.ptr(x), x.stride(0), st), "ezr_embed_gather")
            fp8 = self.precision == "fp8"
            xn = None if fp8 else torch.empty_like(x)         # fp8: the norms write only their e4m3 row
            qkv = torch.empty(t, (H + 2 * KV) * hd, dtype=torch.bfloat16, device=dev)
            ao = torch.empty(t, H * hd, dtype=torch.bfloat16, device=dev)
            act = torch.empty(t, cfg.intermediate_size, dtype=torch.bfloat16, device=dev)
            x8, a8, act8 = (_fp8_dest(b, None, None) if fp8 else None for b in (x, ao, act))
            for ly in self.layers:
                _linear(_norm(x, ly["ln1"], None, cfg.rms_norm_eps, xn, x8), ly["wqkv"], bias=ly["bqkv"], out=qkv)
                _lib.check(L.ezr_rope(_lib.ptr(qkv), qkv.stride(0), _lib.ptr(batch.positions), _lib.ptr(self.cos),
                                      _lib.ptr(self.sin), cfg.max_position_embeddings, H + KV, hd, t, st), "ezr_rope")
                attention(qkv, batch.cu, batch.max_len, H, KV, hd, out=ao, causal=self.causal)
                _linear(_operand(ao, a8), ly["wo"], residual=x, out=x)
                _linear(_norm(x, ly["ln2"], None, cfg.rms_norm_eps, xn, x8), ly["wgu"], out=act, epilogue=EPI_SWIGLU)
                _linear(_operand(act, act8), ly["wdown"], residual=x, out=x)
        return x

    @torch.no_grad()
    def embed_packed(self, batch: PackedBatch, out_bf16: Optional[torch.Tensor] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (bf16 [B, d] unit rows for the dense index, float32 copy the embedding API returns).
        ``out_bf16``: a contiguous [B, d] bf16 destination, e.g. ``DenseIndex.rows_for_append(B)`` -- the pooling
        kernel then writes the corpus rows in place."""
        return _pool(self, batch, out_bf16, POOL_LAST, self.norm, self.cfg.rms_norm_eps, 1)

    def flops(self, lens: Sequence[int]) -> float:
        """SURVEY.md 8(d): layers*(4Ld^2 + 4Ld*kv_dim + 6Ld*ffn + 4L^2 d) per sequence; causal attention counts the
        visible keys only, 2L(L+1)d instead of 4L^2 d."""
        c = self.cfg
        kvd = c.num_key_value_heads * c.head_dim
        att = (lambda n: 2 * n * (n + 1) * c.hidden_size) if self.causal else (lambda n: 4 * n * n * c.hidden_size)
        return float(sum(c.num_hidden_layers * (4 * n * c.hidden_size ** 2 + 4 * n * c.hidden_size * kvd
                                                + 6 * n * c.hidden_size * c.intermediate_size
                                                + att(n)) for n in lens))


# -------------------------------------------------------------------------------------- BERT-shaped
@dataclass
class BertConfig:
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    max_position_embeddings: int = 512
    layer_norm_eps: float = 1e-12

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


class BertEncoder:
    """BERT encoder + CLS/mean pooling + L2 norm == what SentenceTransformer.encode runs for bge-* / gte-base.

    ``state`` uses transformers.BertModel parameter names (``embeddings.*``, ``encoder.layer.N.*``).
    ``precision="fp8"``: the layer GEMMs on e4m3 weights (per-channel scales, no bf16 copy kept) and per-row quantised
    activations, as in Qwen2Encoder; everything else stays bf16.
    """

    def __init__(self, cfg: BertConfig, state: Dict[str, torch.Tensor], device="cuda", pooling: str = "cls",
                 precision: str = "bf16"):
        _check_precision(precision)
        _lib.require_cuda()
        self.cfg = cfg
        self.precision = precision
        self.device = torch.device(device)
        if cfg.head_dim not in (64, 128):
            raise ValueError("head_dim must be 64 or 128")
        self.pool = {"cls": POOL_CLS, "mean": POOL_MEAN, "last": POOL_LAST}[pooling]
        dev = self.device
        g = lambda name: state[name]
        self.word = _bf16(g("embeddings.word_embeddings.weight"), dev)
        self.pos = _bf16(g("embeddings.position_embeddings.weight"), dev)
        self.type_table = _bf16(g("embeddings.token_type_embeddings.weight"), dev)
        self.type0 = self.type_table[0]
        self.emb_g = _bf16(g("embeddings.LayerNorm.weight"), dev)
        self.emb_b = _bf16(g("embeddings.LayerNorm.bias"), dev)
        self.layers = []
        for i in range(cfg.num_hidden_layers):
            p = f"encoder.layer.{i}."
            wqkv = torch.cat([g(p + "attention.self.query.weight"), g(p + "attention.self.key.weight"),
                              g(p + "attention.self.value.weight")], 0)
            bqkv = torch.cat([g(p + "attention.self.query.bias"), g(p + "attention.self.key.bias"),
                              g(p + "attention.self.value.bias")], 0)
            self.layers.append(dict(
                wqkv=_weight(wqkv, dev, precision), bqkv=_bf16(bqkv, dev),
                wo=_weight(g(p + "attention.output.dense.weight"), dev, precision),
                bo=_bf16(g(p + "attention.output.dense.bias"), dev),
                ln1g=_bf16(g(p + "attention.output.LayerNorm.weight"), dev),
                ln1b=_bf16(g(p + "attention.output.LayerNorm.bias"), dev),
                w1=_weight(g(p + "intermediate.dense.weight"), dev, precision),
                b1=_bf16(g(p + "intermediate.dense.bias"), dev),
                w2=_weight(g(p + "output.dense.weight"), dev, precision), b2=_bf16(g(p + "output.dense.bias"), dev),
                ln2g=_bf16(g(p + "output.LayerNorm.weight"), dev), ln2b=_bf16(g(p + "output.LayerNorm.bias"), dev)))

    @torch.no_grad()
    def hidden(self, batch: PackedBatch) -> torch.Tensor:
        L = _lib.lib()
        cfg = self.cfg
        t = batch.ids.numel()
        d, hd, H = cfg.hidden_size, cfg.head_dim, cfg.num_attention_heads
        dev = self.device
        batch.check_positions(cfg.max_position_embeddings)
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            x = torch.empty(t, d, dtype=torch.bfloat16, device=dev)
            if batch.types is None:
                _lib.check(L.ezr_bert_embed(_lib.ptr(batch.ids), _lib.ptr(batch.positions), t, _lib.ptr(self.word),
                                            _lib.ptr(self.pos), _lib.ptr(self.type0), _lib.ptr(self.emb_g),
                                            _lib.ptr(self.emb_b), cfg.layer_norm_eps, cfg.vocab_size,
                                            cfg.max_position_embeddings, d, _lib.ptr(x), st), "ezr_bert_embed")
            else:
                _lib.check(L.ezr_bert_embed_typed(_lib.ptr(batch.ids), _lib.ptr(batch.positions), _lib.ptr(batch.types),
                                                  t, _lib.ptr(self.word), _lib.ptr(self.pos), _lib.ptr(self.type_table),
                                                  self.type_table.shape[0], _lib.ptr(self.emb_g), _lib.ptr(self.emb_b),
                                                  cfg.layer_norm_eps, cfg.vocab_size, cfg.max_position_embeddings, d,
                                                  _lib.ptr(x), st), "ezr_bert_embed_typed")
            qkv = torch.empty(t, 3 * d, dtype=torch.bfloat16, device=dev)
            ao = torch.empty(t, d, dtype=torch.bfloat16, device=dev)
            y = torch.empty(t, d, dtype=torch.bfloat16, device=dev)
            act = torch.empty(t, cfg.intermediate_size, dtype=torch.bfloat16, device=dev)
            x8, a8, act8 = (_fp8_dest(b, None, None) if self.precision == "fp8" else None for b in (x, ao, act))
            h = _operand(x, x8)
            for ly in self.layers:
                # x, the bf16 residual stream, is written by every LayerNorm; h is x as the next GEMM's operand
                _linear(h, ly["wqkv"], bias=ly["bqkv"], out=qkv)
                attention(qkv, batch.cu, batch.max_len, H, H, hd, out=ao)
                _linear(_operand(ao, a8), ly["wo"], bias=ly["bo"], residual=x, out=y)
                h = _norm(y, ly["ln1g"], ly["ln1b"], cfg.layer_norm_eps, x, x8)
                _linear(h, ly["w1"], bias=ly["b1"], out=act, epilogue=EPI_GELU)
                _linear(_operand(act, act8), ly["w2"], bias=ly["b2"], residual=x, out=y)
                h = _norm(y, ly["ln2g"], ly["ln2b"], cfg.layer_norm_eps, x, x8)
        return x

    @torch.no_grad()
    def embed_packed(self, batch: PackedBatch, normalize: bool = True, out_bf16: Optional[torch.Tensor] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor]:
        return _pool(self, batch, out_bf16, self.pool, None, 0.0, 2 if normalize else 0)

    def flops(self, lens: Sequence[int]) -> float:
        """SURVEY.md 8(d): layers*(24 L d^2 + 4 L^2 d) per sequence (ffn = 4d)."""
        c = self.cfg
        per = lambda n: c.num_hidden_layers * (8 * n * c.hidden_size ** 2 + 4 * n * c.hidden_size * c.intermediate_size
                                               + 4 * n * n * c.hidden_size)
        return float(sum(per(n) for n in lens))


def random_state(kind: str, cfg, seed: int, std: float = 0.02) -> Dict[str, torch.Tensor]:
    """Random-init weights of the right shapes (there are no checkpoints offline); values bf16-representable."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *shape, s=std: (torch.randn(*shape, generator=g) * s).to(torch.bfloat16).float()
    st: Dict[str, torch.Tensor] = {}
    d = cfg.hidden_size
    if kind == "qwen2":
        hd, H, KV, ffn = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
        st["embed_tokens.weight"] = rn(cfg.vocab_size, d)
        for i in range(cfg.num_hidden_layers):
            p = f"layers.{i}."
            st[p + "input_layernorm.weight"] = (1 + rn(d, s=0.1))
            st[p + "post_attention_layernorm.weight"] = (1 + rn(d, s=0.1))
            for nm, rows in (("q_proj", H * hd), ("k_proj", KV * hd), ("v_proj", KV * hd)):
                st[p + f"self_attn.{nm}.weight"] = rn(rows, d)
                st[p + f"self_attn.{nm}.bias"] = rn(rows)
            st[p + "self_attn.o_proj.weight"] = rn(d, H * hd)
            st[p + "mlp.gate_proj.weight"] = rn(ffn, d)
            st[p + "mlp.up_proj.weight"] = rn(ffn, d)
            st[p + "mlp.down_proj.weight"] = rn(d, ffn)
        st["norm.weight"] = (1 + rn(d, s=0.1))
    elif kind == "bert":
        ffn = cfg.intermediate_size
        st["embeddings.word_embeddings.weight"] = rn(cfg.vocab_size, d)
        st["embeddings.position_embeddings.weight"] = rn(cfg.max_position_embeddings, d)
        st["embeddings.token_type_embeddings.weight"] = rn(2, d)
        st["embeddings.LayerNorm.weight"] = 1 + rn(d, s=0.1)
        st["embeddings.LayerNorm.bias"] = rn(d)
        for i in range(cfg.num_hidden_layers):
            p = f"encoder.layer.{i}."
            for nm in ("query", "key", "value"):
                st[p + f"attention.self.{nm}.weight"] = rn(d, d)
                st[p + f"attention.self.{nm}.bias"] = rn(d)
            st[p + "attention.output.dense.weight"] = rn(d, d)
            st[p + "attention.output.dense.bias"] = rn(d)
            st[p + "attention.output.LayerNorm.weight"] = 1 + rn(d, s=0.1)
            st[p + "attention.output.LayerNorm.bias"] = rn(d)
            st[p + "intermediate.dense.weight"] = rn(ffn, d)
            st[p + "intermediate.dense.bias"] = rn(ffn)
            st[p + "output.dense.weight"] = rn(d, ffn)
            st[p + "output.dense.bias"] = rn(d)
            st[p + "output.LayerNorm.weight"] = 1 + rn(d, s=0.1)
            st[p + "output.LayerNorm.bias"] = rn(d)
    else:
        raise ValueError(kind)
    return st
