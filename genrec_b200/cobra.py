"""COBRA (SURVEY.md section 8): drop-in mirror of ``genrec/models/cobra.py:47-529`` for training, with its ``LightT5Encoder``
(``genrec/modules/encoder.py:15-105``).

Same constructor arguments, parameter and buffer names / shapes (a reference checkpoint loads with ``strict=True``), ``forward``
-> ``CobraOutput`` and ``generate_itemvec`` as the reference's ``Cobra``; ``encode_items`` adds the catalog vectors BeamFusion needs.
Bind it with

    import genrec.models.cobra, genrec_b200.cobra
    genrec.models.cobra.Cobra = genrec_b200.cobra.Cobra

Item-text encoder: the texts are packed into token rows on the device (``functional.cobra_pack_texts``): a text is its leading
non-zero tokens and the texts of pad items have none, so neither text pads nor pad items are encoded (the reference's key mask and
pooling keep both out of every output).  A text where a non-zero token follows a zero is refused with ValueError.  The projections
and the ReLU FFN are the wgmma GEMMs of this library (ReLU and the hidden dropout in the GEMM epilogue, the output dropout and the
residual in the second GEMM's), attention is the packed T5 core at head dim 96 (no bias, not causal), the post-LN residual norms
the LayerNorm row kernels, the final LayerNorm and the mean over each text one segmented kernel, then the ``proj`` GEMM and an L2
normalisation kernel.

Decoder: the interleaved [sparse ids of item t, dense vector of item t] sequence (torch gathers), self-attention on the padded T5
core (causal, key padding, no bias), the cross-attention over the empty memory as the bias add it reduces to (its projection
weights get zero gradients, as in the reference), post-LN and the ReLU FFN as in the encoder.

Heads: three 384 -> 256 GEMMs on their gathered rows with a cross-entropy in torch (ignore_index = pad_id); the in-batch InfoNCE
is a GEMM for the scores, one row kernel for the loss and dS, and a GEMM for dpred.  bf16 operands, fp32 accumulation.  The
embedding gathers, the residual adds, the dropouts on the residual branches and the metrics stay in torch.  Dropout seeds come
from torch's CPU generator, so ``torch.manual_seed`` makes a step reproducible bit for bit.

Generation (``generate``, cobra.py:531-665) decodes each user's history once: the encoder and the decoder run over the B padded
histories (``_decode``, which keeps every layer's QKV), and each later codebook is one new token per beam.  Its layer runs the QKV
GEMM into a per-step buffer, ``grb_cobra_beam_attention`` (the history's K | V read in place from the prefill's QKV, the beam's own
earlier tokens through an ancestry table), and then the same layer body as training (``_layer_tail``).  ``grb_cobra_beam_topk``
adds log_softmax(logits / temperature) to the parents' scores and keeps the K best per user, writing the next ancestry table, so
beam selection never moves K | V.  Each user gets the beams the reference gives that user alone (INTEGRATION.md), bit for bit
whatever the batch around it.  ``beam_fusion`` (cobra.py:679-760) finds each beam's best catalog row with ``grb_cobra_dense_match``,
one wgmma sweep of the bf16 catalog, without the [B, n_beam, N] similarity; the B x n_beam fusion tail stays in torch.  Both run
without gradients and without dropout, and read two values to the host: the item-layout flag of ``_check_generate`` and the
encoder's packing info.

Serving (``new_pool`` -> ``CobraPool``, ``extend_users``, ``generate_users``, ``beam_fusion_users``, ``CobraPool.release``): every
decoder layer's K | V rows of many users live in one paged pool.  ``extend_users`` encodes only the new items' texts and runs only
their decoder rows, at the positions that continue each user's history: per layer the QKV GEMM, ``grb_cobra_kv_scatter`` (the new
K | V rows into the user's pages), ``grb_cobra_paged_attention`` (each new row against everything the user has cached, read from the
pages) and ``_layer_tail``; the final layer's row at the last dense position is kept as the user's ``last_hidden``.
``generate_users`` runs ``generate``'s beam search (``_beams``, shared) from ``last_hidden`` with the history read through the page
table.  The host keeps every user's item count and pages, so every refusal comes before any launch.  A user's outputs are the same
bits however the history was split into calls and whichever users share the call or the pool.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from . import functional as Fn
from ._lib import ensure_device, require_cuda
from .t5_attention import attention_core_bwd, attention_core_bwd_jagged, attention_core_fwd, attention_core_fwd_jagged

__all__ = ["Cobra", "CobraOutput", "CobraGenerationOutput", "BeamFusionOutput", "CobraPool"]

LN_DIMS = (64, 128, 192, 256, 384, 768)           # widths of the LayerNorm row kernels
POOL_DIMS = (128, 192, 256, 384, 768)             # widths of the pooled LayerNorm kernel
ENC_HEAD_DIMS = (32, 64, 96)
DEC_HEAD_DIMS = (32, 64)
MAX_ATTN_ROWS = 65535                             # texts x heads (or users x heads) of one attention backward
_MAX_BEAMS = 1024                                 # beams per user of generate (grb_cobra_beam_topk, grb_cobra_beam_attention)
_MAX_CANDIDATES = 262144                          # beams x id_vocab_size of one beam step
_CATALOG_CHUNK = 65536                            # catalog rows normalised at a time by beam_fusion
_MAX_KEYS = 8192                                  # history rows of one user in the beam attention (CBA_MAX_HIST)


class CobraGenerationOutput(NamedTuple):     # (cobra.py:29-35)
    sem_ids: torch.Tensor           # [B, K, C]
    dense_vecs: torch.Tensor        # [B, K, d_model]
    scores: torch.Tensor            # [B, K]


class BeamFusionOutput(NamedTuple):          # (cobra.py:38-44)
    item_ids: torch.Tensor          # [B, K]
    sem_ids: torch.Tensor           # [B, K, C]
    scores: torch.Tensor            # [B, K]


class _MissingArguments(TypeError, NotImplementedError):
    """a generation call without its history inputs: a TypeError naming them, as Python's own, and a NotImplementedError, which a
    call without arguments raised before generation was native"""

    def __init__(self, fn: str, names):
        super().__init__(f"{fn}() missing {len(names)} required argument{'s' if len(names) > 1 else ''}: "
                         + ", ".join(repr(n) for n in names))


class CobraOutput(NamedTuple):      # (cobra.py:12-26)
    loss: torch.Tensor
    loss_sparse: torch.Tensor
    loss_dense: torch.Tensor
    acc_correct: torch.Tensor
    acc_total: torch.Tensor
    recall_correct: torch.Tensor
    recall_total: torch.Tensor
    vec_cos_sim: torch.Tensor
    codebook_entropy: torch.Tensor


class CobraPool:
    """Paged per-user decoder cache of ``Cobra`` for serving (``Cobra.new_pool`` / ``extend_users`` / ``generate_users`` /
    ``beam_fusion_users`` / ``CobraPool.release``).

    Every decoder layer's K | V rows live in ``num_pages`` pages of ``page_size`` decoder positions shared by all users (``kv``
    [decoder_layers, num_pages, page_size, 2 d_model] bf16); ``page_table`` [max_users, ceil(max_items (C+1) / page_size)] int32 maps
    user u's position p to page ``page_table[u, p // page_size]`` (entries past a user's pages are 0).  ``last_hidden`` [max_users,
    d_model] fp32 is each user's final-layer row at their last dense position, where ``generate_users`` starts.  The host keeps each
    user's exact item count (``lengths``) and page list, and the free pages as a stack (page 0 goes out first): a call takes the pages
    it needs in row order, and ``release`` pushes a user's pages back, first page on top.

    A pool belongs to the parameters it was first written with: a later call raises once any parameter's version counter has moved
    (a torch optimizer step, ``load_state_dict``).  ``genrec_b200.optim.FlatAdam`` writes parameters through a raw pointer and is not
    caught, so rebuild every pool after any further training.
    """

    def __init__(self, max_users: int, num_pages: int, page_size: int, max_items: int, num_layers: int, d_model: int, C: int, device):
        self.max_users, self.num_pages, self.page_size, self.max_items, self.C = max_users, num_pages, page_size, max_items, C
        self.kv = torch.zeros(num_layers, num_pages, page_size, 2 * d_model, dtype=torch.bfloat16, device=device)
        self.page_table = torch.zeros(max_users, -(-max_items * (C + 1) // page_size), dtype=torch.int32, device=device)
        self.last_hidden = torch.zeros(max_users, d_model, dtype=torch.float32, device=device)
        self.lengths = [0] * max_users                # items per user (host)
        self.pages = [[] for _ in range(max_users)]   # each user's pages in position order (host)
        self.free = list(range(num_pages - 1, -1, -1))
        self.param_versions = None

    def pages_free(self) -> int:
        return len(self.free)

    def _users(self, users, fn: str) -> list:
        u = (users if isinstance(users, torch.Tensor) else torch.as_tensor(users)).reshape(-1).tolist()
        if not u or not all(isinstance(x, int) for x in u):
            raise ValueError(f"{fn}: users must be a non-empty list of integers, got {users!r}")
        bad = [x for x in u if not 0 <= x < self.max_users]
        if bad:
            raise ValueError(f"{fn}: users out of range [0, {self.max_users}): {bad[:8]}")
        if len(set(u)) != len(u):
            raise ValueError(f"{fn}: users must be distinct within a call")
        return u

    def _pages_for(self, items: int) -> int:
        return -(-items * (self.C + 1) // self.page_size)

    def release(self, users) -> None:
        """Forget ``users`` (distinct, any subset): their pages return to the pool, their lengths and ``last_hidden`` become zero,
        and the next ``extend_users`` starts their histories afresh."""
        u = self._users(users, "CobraPool.release")
        for x in u:
            self.free.extend(reversed(self.pages[x]))
            self.pages[x] = []
            self.lengths[x] = 0
        idx = torch.tensor(u, dtype=torch.int64).to(self.kv.device)
        self.page_table.index_fill_(0, idx, 0)
        self.last_hidden.index_fill_(0, idx, 0.0)


def _bad(msg: str) -> _lib.GrbError:
    return _lib.GrbError(f"genrec_b200 error -1: {msg}")


# ---- autograd pieces
class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, g, b, eps):
        xc = x.detach().contiguous().float()
        y, st = Fn.post_layernorm_fwd(xc, g.detach().contiguous(), b.detach().contiguous(), eps)
        ctx.save_for_backward(xc, st, g)
        return y

    @staticmethod
    def backward(ctx, dy):
        xc, st, g = ctx.saved_tensors
        dx, dg, db = Fn.post_layernorm_bwd(dy.contiguous().float(), xc, st, g.detach().contiguous())
        return dx, dg, db, None


class _LinearF32Fn(torch.autograd.Function):
    """nn.Linear with an fp32 result: y = x W^T + b (the GEMM writes fp32, the bias is added in fp32)."""

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.empty = x.numel() == 0                    # no rows (no user has a second item): nothing to launch
        if ctx.empty:
            ctx.shapes = (x.shape, w.shape)
            return x.new_zeros(*x.shape[:-1], w.shape[0], dtype=torch.float32)
        xb = Fn.cast_rows_bf16(x.detach().contiguous().float())
        wb = Fn.cast_bf16(w)
        ctx.save_for_backward(xb, wb)
        return Fn.matmul_f32(xb, wb.t().contiguous()) + b.detach()

    @staticmethod
    def backward(ctx, dy):
        if ctx.empty:
            xs, ws = ctx.shapes
            return dy.new_zeros(xs), dy.new_zeros(ws), dy.new_zeros(ws[0])
        xb, wb = ctx.saved_tensors
        dyc = dy.contiguous().float()
        dx, dw, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dyc), wb, xb)
        return dx, dw, dyc.reshape(-1, dyc.shape[-1]).sum(0)


class _MhaFn(torch.autograd.Function):
    """nn.MultiheadAttention self-attention (in_proj with bias, out_proj with bias) on the T5 core without a bias table.  Padded:
    x [B, L, D] with key_pad [B, L] uint8 and causal; packed: x [T, D] with offsets [N+1] and max_len (no key padding)."""

    @staticmethod
    def forward(ctx, x, w_in, b_in, w_out, b_out, H, p, seed, site, key_pad, causal, offsets, max_len, keep_qkv=None):
        D = x.shape[-1]
        xb = Fn.cast_rows_bf16(x.detach().contiguous().float())
        wib, wob = Fn.cast_bf16(w_in), Fn.cast_bf16(w_out)
        QKV, _ = Fn.linear_fwd(xb, wib, b_in.detach().contiguous(), 0)
        if keep_qkv is not None:                      # generation's prefill keeps every layer's K | V
            keep_qkv.append(QKV)
        Q, K, V = QKV[..., :D], QKV[..., D:2 * D], QKV[..., 2 * D:]
        scale = 1.0 / math.sqrt(D // H)
        if offsets is None:
            A, lse = attention_core_fwd(Q, K, V, H, None, None, key_pad, causal, scale, p, seed, site)
        else:
            A, lse = attention_core_fwd_jagged(Q, K, V, H, None, None, offsets, max_len, causal, scale, p, seed, site)
        out, _ = Fn.linear_fwd(A, wob, b_out.detach().contiguous(), 0)
        ctx.save_for_backward(xb, QKV, A, lse, wib, wob, key_pad if key_pad is not None else lse, offsets if offsets is not None else lse)
        ctx.cfg = (H, p, seed, site, scale, causal, key_pad is not None, offsets is not None, max_len)
        return out.float()

    @staticmethod
    def backward(ctx, dout):
        xb, QKV, A, lse, wib, wob, key_pad, offsets = ctx.saved_tensors
        H, p, seed, site, scale, causal, has_pad, packed, max_len = ctx.cfg
        D = A.shape[-1]
        Q, K, V = QKV[..., :D], QKV[..., D:2 * D], QKV[..., 2 * D:]
        dA, dwo, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dout.contiguous().float()), wob, A)
        dAb = Fn.cast_rows_bf16(dA)
        if packed:
            dQ, dK, dV, _ = attention_core_bwd_jagged(Q, K, V, H, None, None, offsets, max_len, causal, scale, A, lse, dAb, p, seed, site)
        else:
            dQ, dK, dV, _ = attention_core_bwd(Q, K, V, H, None, None, key_pad if has_pad else None, causal, scale, A, lse, dAb, p, seed,
                                               site)
        dqkv = torch.cat([dQ.float(), dK, dV], dim=-1)
        dx, dwi, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dqkv), wib, xb)
        dyc = dout.contiguous().float()
        return (dx, dwi, dqkv.reshape(-1, 3 * D).sum(0), dwo, dyc.reshape(-1, D).sum(0), None, None, None, None, None, None, None, None,
                None)


class _FfnFn(torch.autograd.Function):
    """x + drop(linear2(drop(relu(linear1(x))))) with biases: ReLU and the hidden dropout in the first GEMM's epilogue, the output
    dropout and the residual in the second's."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, p_in, p_out, seed, site):
        xc = x.detach().contiguous().float()
        xb = Fn.cast_rows_bf16(xc)
        w1b, w2b = Fn.cast_bf16(w1), Fn.cast_bf16(w2)
        y, z, h = Fn.ffn_fwd(xb, w1b, b1.detach().contiguous(), w2b, b2.detach().contiguous(), xc, None, p_in, p_out, seed, None, site,
                             site + 1)
        ctx.save_for_backward(xb, z, h, w1b, w2b)
        ctx.cfg = (p_in, p_out, seed, site)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, z, h, w1b, w2b = ctx.saved_tensors
        p_in, p_out, seed, site = ctx.cfg
        dyc = dy.contiguous().float()
        dx, dw1, db1, dw2, db2 = Fn.ffn_bwd(dyc, w1b, w2b, xb, z, h, p_in, p_out, seed, None, site, site + 1, dx_residual=dyc)
        return dx, dw1, db1, dw2, db2, None, None, None, None


class _SegLnMeanFn(torch.autograd.Function):
    """pooled [N, D] = mean over the rows of each text of LayerNorm(x) (encoder.py:88-96 on packed rows)"""

    @staticmethod
    def forward(ctx, x, g, b, offsets, eps):
        xc = x.detach().contiguous().float()
        pooled, st = Fn.seg_layernorm_mean_fwd(offsets, xc, g.detach().contiguous(), b.detach().contiguous(), eps)
        ctx.save_for_backward(xc, st, g, offsets)
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        xc, st, g, offsets = ctx.saved_tensors
        dx, dg, db = Fn.seg_layernorm_mean_bwd(offsets, xc, st, g.detach().contiguous(), dpooled.contiguous().float())
        return dx, dg, db, None, None


class _L2NormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, n = Fn.l2norm_fwd(x.detach().contiguous().float())
        ctx.save_for_backward(y, n)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, n = ctx.saved_tensors
        return Fn.l2norm_bwd(dy.contiguous().float(), y, n)


class _InfoNceFn(torch.autograd.Function):
    """mean over the Q rows of the in-batch InfoNCE of unit rows pred, gt [Q, d] (cobra.py:484-493); no gradient into gt"""

    @staticmethod
    def forward(ctx, pred, gt, lo, hi, inv_tau):
        Q, d = pred.shape
        Qp = (Q + 127) // 128 * 128                  # dS is the K operand of the dpred GEMM: at least two 64-wide K tiles
        pb = Fn.cast_rows_bf16(pred.detach().contiguous())
        gpad = torch.zeros(Qp, d, dtype=torch.bfloat16, device=pred.device)
        gpad[:Q] = Fn.cast_rows_bf16(gt.detach().contiguous())
        S = Fn.matmul_f32(pb, gpad.t().contiguous())                                # [Q, Qp] = pred gt^T
        loss, dS = Fn.infonce_fwd_bwd(S, lo, hi, inv_tau)
        ctx.save_for_backward(dS, gpad)
        return (loss / Q).reshape(())

    @staticmethod
    def backward(ctx, g):
        dS, gpad = ctx.saved_tensors
        return Fn.matmul_f32(dS, gpad) * g, None, None, None, None


class _ZeroGrads(torch.autograd.Function):
    """t unchanged; the other inputs get zero-tensor gradients (the cross-attention weights that an empty memory never reaches, and
    the encoder when no text has a token: the reference's autograd gives them zero tensors, not None, which AdamW's weight decay
    tells apart)."""

    @staticmethod
    def forward(ctx, t, *others):
        ctx.shapes = [(o.shape, o.dtype, o.device) for o in others]
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return (g, *[torch.zeros(s, dtype=dt, device=dev) for s, dt, dev in ctx.shapes])


# ---- modules with the reference's parameter names (encoder.py:15-60, cobra.py:47-224)
class _LightT5Encoder(nn.Module):
    def __init__(self, n_layers, hidden_dim, output_dim, num_heads, ff_dim=2048, vocab_size=32128, max_seq_len=512, dropout=0.1):
        super().__init__()
        self.embedding = nn.Embedding(vocab_size, hidden_dim)
        self.pos_embedding = nn.Embedding(max_seq_len, hidden_dim)
        layer = nn.TransformerEncoderLayer(d_model=hidden_dim, nhead=num_heads, dim_feedforward=ff_dim, dropout=dropout, batch_first=True)
        self.encoder = nn.TransformerEncoder(layer, num_layers=n_layers, enable_nested_tensor=False)
        self.proj = nn.Linear(hidden_dim, output_dim)
        self.layer_norm = nn.LayerNorm(hidden_dim)


class _CobraEmbedding(nn.Module):
    def __init__(self, id_vocab_size, n_codebooks=3, d_model=768, max_len=1024, pad_id=0):
        super().__init__()
        self.C, self.pad_id, self.id_vocab_size = n_codebooks, pad_id, id_vocab_size
        self.id_embed = nn.Embedding(id_vocab_size * n_codebooks + 1, d_model, padding_idx=id_vocab_size * n_codebooks)
        self.type_embed = nn.Embedding(2, d_model)
        self.pos_embed = nn.Embedding(max_len, d_model)


class _CobraDecoder(nn.Module):
    def __init__(self, hidden_dim, n_layers, n_heads, ff_dim=2048, dropout=0.1):
        super().__init__()
        layer = nn.TransformerDecoderLayer(d_model=hidden_dim, nhead=n_heads, dim_feedforward=ff_dim, dropout=dropout, batch_first=True)
        self.decoder = nn.TransformerDecoder(layer, num_layers=n_layers)


class Cobra(nn.Module):
    """Mirror of genrec/models/cobra.py:227-529 (training and item vectors)."""

    def __init__(self, encoder_n_layers: int = 1, encoder_hidden_dim: int = 768, encoder_num_heads: int = 8, encoder_vocab_size: int = 32128,
                 id_vocab_size: int = 512, n_codebooks: int = 3, d_model: int = 768, max_len: int = 1024, temperature=0.2, queue_size=1024,
                 decoder_n_layers: int = 8, decoder_num_heads: int = 6, decoder_dropout: float = 0.1, encoder_type: str = "light",
                 encoder_model_name: str = "./models_hub/sentence-t5-base") -> None:
        super().__init__()
        if encoder_type != "light":
            raise NotImplementedError("genrec_b200.Cobra: only the light (randomly initialised) item-text encoder is native")
        if encoder_hidden_dim not in POOL_DIMS or encoder_hidden_dim % encoder_num_heads or \
                encoder_hidden_dim // encoder_num_heads not in ENC_HEAD_DIMS:
            raise _bad(f"encoder_hidden_dim {encoder_hidden_dim} with {encoder_num_heads} heads unsupported (widths {POOL_DIMS}, "
                       f"head dims {ENC_HEAD_DIMS})")
        if d_model not in LN_DIMS or d_model % decoder_num_heads or d_model // decoder_num_heads not in DEC_HEAD_DIMS:
            raise _bad(f"d_model {d_model} with {decoder_num_heads} heads unsupported (widths {LN_DIMS}, head dims {DEC_HEAD_DIMS})")
        self.C = n_codebooks
        self.d_model = d_model
        self.pad_id = id_vocab_size * self.C
        self.max_len = max_len
        self.encoder = _LightT5Encoder(n_layers=encoder_n_layers, hidden_dim=encoder_hidden_dim, output_dim=d_model,
                                       num_heads=encoder_num_heads, vocab_size=encoder_vocab_size)
        self.cobra_emb = _CobraEmbedding(id_vocab_size=id_vocab_size, d_model=d_model, max_len=max_len, pad_id=self.pad_id)
        self.decoder = _CobraDecoder(d_model, n_layers=decoder_n_layers, n_heads=decoder_num_heads, dropout=decoder_dropout)
        self.sparse_head = nn.ModuleList([nn.Linear(d_model, id_vocab_size) for _ in range(n_codebooks)])
        self.temperature = temperature
        self.register_buffer("feat_queue", torch.randn(queue_size, d_model))
        self.register_buffer("queue_ptr", torch.zeros(1, dtype=torch.long))
        self.queue_size = queue_size
        self.feat_queue = F.normalize(self.feat_queue, dim=-1)

    # ---- dropout
    def _p(self, p: float) -> float:
        return p if self.training else 0.0

    def _drop(self, x, p):
        return F.dropout(x, p, self.training) if self.training and p > 0 else x

    def _seed(self) -> int:
        """one dropout seed per step from torch's CPU generator (reproducible under torch.manual_seed, new every step)"""
        return int(torch.randint(1, 1 << 62, (1,)).item()) if self.training else 0

    # ---- item-text encoder
    def _encode(self, tokens: torch.Tensor, keep: Optional[torch.Tensor]) -> torch.Tensor:
        """tokens [N, L] -> normalised item vectors [N, d_model] fp32 (encoder.py:61-103 on packed rows)"""
        require_cuda(tokens)
        ensure_device(tokens.device)
        enc = self.encoder
        N, L = tokens.shape
        if L > enc.pos_embedding.num_embeddings:
            raise _bad(f"text length {L} exceeds the position table ({enc.pos_embedding.num_embeddings})")
        tokens = tokens.contiguous().long()
        offsets, info = Fn.cobra_pack_texts(tokens, keep)
        rows, longest, bad = info.tolist()
        if bad:
            raise ValueError(f"Cobra: text {bad - 1} has a non-zero token after a zero; item texts must be right-padded with 0")
        H = enc.encoder.layers[0].self_attn.num_heads
        if torch.is_grad_enabled() and N * H > MAX_ATTN_ROWS:
            raise _bad(f"{N} texts x {H} heads exceed {MAX_ATTN_ROWS} for the attention backward")
        hid = enc.embedding.embedding_dim
        if rows == 0:
            # no text has a token: every pooled vector is zero.  The reference still runs the encoder, whose parameters (all but
            # proj) get zero-tensor gradients through the masked pooling; they get the same here, so AdamW decays them alike.
            skipped = [p for n, p in enc.named_parameters() if not n.startswith("proj.")]
            pooled = _ZeroGrads.apply(torch.zeros(N, hid, dtype=torch.float32, device=tokens.device), *skipped)
        else:
            tok, pos = Fn.cobra_text_rows(tokens, offsets, rows)
            x = F.embedding(tok, enc.embedding.weight) + F.embedding(pos, enc.pos_embedding.weight)
            seed = self._seed()
            for i, layer in enumerate(enc.encoder.layers):
                sa = layer.self_attn
                a = _MhaFn.apply(x, sa.in_proj_weight, sa.in_proj_bias, sa.out_proj.weight, sa.out_proj.bias, sa.num_heads,
                                 self._p(sa.dropout), seed, 16 * i + 1, None, False, offsets, longest)
                x = _LayerNormFn.apply(x + self._drop(a, layer.dropout1.p), layer.norm1.weight, layer.norm1.bias, layer.norm1.eps)
                f = _FfnFn.apply(x, layer.linear1.weight, layer.linear1.bias, layer.linear2.weight, layer.linear2.bias,
                                 self._p(layer.dropout.p), self._p(layer.dropout2.p), seed, 16 * i + 2)
                x = _LayerNormFn.apply(f, layer.norm2.weight, layer.norm2.bias, layer.norm2.eps)
            pooled = _SegLnMeanFn.apply(x, enc.layer_norm.weight, enc.layer_norm.bias, offsets, enc.layer_norm.eps)
        return _L2NormFn.apply(_LinearF32Fn.apply(pooled, enc.proj.weight, enc.proj.bias))

    def encode_items(self, tokens: torch.Tensor) -> torch.Tensor:
        """Catalog vectors for BeamFusion (the reference's compute_item_dense_vecs): tokens [N, L] -> [N, d_model], each the
        normalised encoder vector of its text (what generate_itemvec gives for the same texts)."""
        return _L2NormFn.apply(self._encode(tokens, None))

    def generate_itemvec(self, encoder_input_ids: torch.Tensor):
        """cobra.py:667-677"""
        if encoder_input_ids.dim() == 3:
            B, T, L = encoder_input_ids.shape
            return self.encode_items(encoder_input_ids.reshape(B * T, L)).view(B, T, -1)
        if encoder_input_ids.dim() != 2:
            raise ValueError(f"Expected 2D or 3D input, got {encoder_input_ids.dim()}D")
        return self.encode_items(encoder_input_ids)

    # ---- decoder
    def _interleave(self, input_ids, vecs, mask_items, start=None):
        """CobraEmbedding.forward (cobra.py:75-147) for complete items: -> (h [B, T(C+1), d] fp32, mask [B, T(C+1)] bool); start [B]
        int64: the decoder position of each row's first item (None: 0)"""
        e = self.cobra_emb
        B, L = input_ids.shape
        C, T = self.C, L // self.C
        dev = input_ids.device
        ct = torch.arange(L, device=dev) % C
        ids = torch.where(input_ids != self.pad_id, input_ids + ct * e.id_vocab_size, input_ids)
        tok = F.embedding(ids, e.id_embed.weight, padding_idx=e.id_embed.padding_idx)
        h = torch.cat([tok.view(B, T, C, -1), vecs.view(B, T, 1, -1)], dim=2).reshape(B, T * (C + 1), -1)
        mask = torch.cat([mask_items, mask_items[:, :, C - 1:]], dim=2).reshape(B, T * (C + 1))
        Li = T * (C + 1)
        types = torch.arange(Li, device=dev) % (C + 1) == C
        m = mask.unsqueeze(-1).float()
        if start is None:
            pos = e.pos_embed.weight[:Li].unsqueeze(0)
        else:                                         # positions past the table only on pad rows, which m zeroes
            pos = e.pos_embed.weight[(start[:, None] + torch.arange(Li, device=dev)).clamp_max(e.pos_embed.num_embeddings - 1)]
        h = h * m + pos * m + F.embedding(types.long(), e.type_embed.weight).unsqueeze(0) * m
        return h, mask

    def _decode(self, x, mask, keep_qkv=None):
        """keep_qkv: a list that receives each layer's self-attention QKV [B, Li, 3D] bf16 (generation's prefill), or None"""
        key_pad = (~mask).to(torch.uint8).contiguous()
        seed = self._seed()
        for i, layer in enumerate(self.decoder.decoder.layers):
            sa = layer.self_attn
            a = _MhaFn.apply(x, sa.in_proj_weight, sa.in_proj_bias, sa.out_proj.weight, sa.out_proj.bias, sa.num_heads, self._p(sa.dropout),
                             seed, 16 * i + 1, key_pad, True, None, 0, keep_qkv)
            x = self._layer_tail(i, layer, x, a, seed)
        return x

    def _layer_tail(self, i, layer, x, a, seed):
        """a decoder layer after its self-attention output a: the residual and norm1, the cross-attention and norm2, the FFN and norm3"""
        ca = layer.multihead_attn
        x = _LayerNormFn.apply(x + self._drop(a, layer.dropout1.p), layer.norm1.weight, layer.norm1.bias, layer.norm1.eps)
        # attention over a zero-length memory is the out_proj bias (cobra.py:209-223)
        cross = _ZeroGrads.apply(ca.out_proj.bias, ca.in_proj_weight, ca.in_proj_bias, ca.out_proj.weight).expand_as(x)
        x = _LayerNormFn.apply(x + self._drop(cross, layer.dropout2.p), layer.norm2.weight, layer.norm2.bias, layer.norm2.eps)
        f = _FfnFn.apply(x, layer.linear1.weight, layer.linear1.bias, layer.linear2.weight, layer.linear2.bias, self._p(layer.dropout.p),
                         self._p(layer.dropout3.p), seed, 16 * i + 2)
        return _LayerNormFn.apply(f, layer.norm3.weight, layer.norm3.bias, layer.norm3.eps)

    # ---- the reference's interface
    def forward(self, input_ids: torch.Tensor, encoder_input_ids: torch.Tensor, mask=None) -> CobraOutput:
        """cobra.py:379-529.  input_ids [B, T*C], encoder_input_ids [B, T, L] (right-padded with 0)."""
        require_cuda(input_ids, encoder_input_ids)
        B, TC = input_ids.shape
        C = self.C
        if TC % C or encoder_input_ids.dim() != 3 or encoder_input_ids.shape[:2] != (B, TC // C):
            raise ValueError(f"Cobra.forward: input_ids [B, T*C] and encoder_input_ids [B, T, L] expected, got {tuple(input_ids.shape)} "
                             f"and {tuple(encoder_input_ids.shape)}")
        T = TC // C
        if T * (C + 1) > self.max_len:
            raise _bad(f"interleaved length {T * (C + 1)} exceeds max_len {self.max_len}")
        H = self.decoder.decoder.layers[0].self_attn.num_heads
        if torch.is_grad_enabled() and B * H > MAX_ATTN_ROWS:
            raise _bad(f"{B} users x {H} heads exceed {MAX_ATTN_ROWS} for the attention backward")
        L = encoder_input_ids.shape[2]
        mask_items = (input_ids != self.pad_id).view(B, T, C)
        keep = mask_items[:, :, C - 1].reshape(-1).to(torch.uint8).contiguous()      # pad items: no rows
        vecs = self._encode(encoder_input_ids.reshape(B * T, L), keep).view(B, T, -1)
        emb, seq_mask = self._interleave(input_ids, vecs, mask_items)
        h = self._decode(emb, seq_mask)
        dev = h.device

        loss_sparse = 0.0
        total_correct = total_tokens = 0
        all_item_correct = torch.ones(B, T - 1, dtype=torch.bool, device=dev)
        all_valid_mask = None
        for c in range(C):                                                         # cobra.py:417-457
            if c == 0:
                pos_c = torch.arange(0, T - 1, device=dev) * (C + 1) + C
                target = input_ids[:, torch.arange(1, T, device=dev) * C]
            else:
                pos_c = torch.arange(1, T, device=dev) * (C + 1) + (c - 1)
                target = input_ids[:, torch.arange(1, T, device=dev) * C + c]
            head = self.sparse_head[c]
            logits = _LinearF32Fn.apply(h[:, pos_c, :], head.weight, head.bias)
            loss_c = F.cross_entropy(logits.reshape(-1, logits.size(-1)), target.reshape(-1), ignore_index=self.pad_id, reduction="sum")
            loss_sparse = loss_sparse + loss_c / (target != self.pad_id).sum().clamp(min=1)
            with torch.no_grad():
                valid_mask = target != self.pad_id
                if all_valid_mask is None:
                    all_valid_mask = valid_mask
                pred_top1 = logits.argmax(-1)
                total_correct = total_correct + ((pred_top1 == target) & valid_mask).sum()
                total_tokens = total_tokens + valid_mask.sum()
                all_item_correct &= (pred_top1 == target) | ~valid_mask
        loss_sparse = loss_sparse / C
        item_correct_masked = all_item_correct & all_valid_mask

        # dense InfoNCE (cobra.py:466-493): rows grouped by user, each user's other items left out
        vec_pos = torch.arange(1, T, device=dev) * (C + 1) + (C - 1)
        valid = seq_mask[:, (C + 1)::(C + 1)]                                       # [B, T-1]
        vec_pred = h[:, vec_pos, :self.d_model][valid]
        vec_gt = Fn.l2norm_fwd(vecs[:, 1:].detach()[valid].contiguous())[0] if vec_pred.shape[0] else vec_pred.detach()
        Q = vec_pred.shape[0]
        if Q == 0:
            loss_dense = vec_cos_sim = torch.full((), float("nan"), device=dev)     # an empty cross-entropy's mean
        else:
            vec_pred = _L2NormFn.apply(vec_pred)
            counts = valid.sum(1)
            ends = counts.cumsum(0)
            user = torch.arange(B, device=dev).repeat_interleave(counts, output_size=Q)
            hi = ends[user]
            lo = hi - counts[user]
            loss_dense = _InfoNceFn.apply(vec_pred, vec_gt, lo.contiguous(), hi.contiguous(), 1.0 / self.temperature)
            with torch.no_grad():
                vec_cos_sim = F.cosine_similarity(vec_pred, vec_gt).mean()
        with torch.no_grad():                                                      # cobra.py:514-517, stride 3 as written
            usage = torch.stack([F.one_hot(input_ids[:, c::3], self.pad_id + 1).sum((0, 1)).float() for c in range(C)])
            prob = usage / usage.sum(1, keepdim=True)
            codebook_entropy = -(prob * (prob.add(1e-12).log())).sum(1).mean()
        return CobraOutput(loss=loss_sparse + loss_dense, loss_sparse=loss_sparse, loss_dense=loss_dense, acc_correct=total_correct,
                           acc_total=total_tokens, recall_correct=item_correct_masked.sum(), recall_total=all_valid_mask.sum(),
                           vec_cos_sim=vec_cos_sim, codebook_entropy=codebook_entropy)

    # ---- generation (cobra.py:531-760)
    def generate(self, input_ids: Optional[torch.Tensor] = None, encoder_input_ids: Optional[torch.Tensor] = None, n_candidates: int = 10,
                 temperature: float = 1.0) -> CobraGenerationOutput:
        """cobra.py:531-665 with per-user semantics: each user gets the beams the reference gives that user alone (its generated token j
        at position n_b (C+1) + j, attending to its own n_b (C+1) history rows), whatever the batch around it.  input_ids [B, T*C] with
        pad items after the real ones, encoder_input_ids [B, T, L] right-padded with 0.  -> sem_ids [B, K, C], dense_vecs [B, K, d_model]
        (unit rows of h at the last input position of the final step), scores [B, K] (summed log-softmax of logits / temperature), best
        first, equal totals by the lower beam * V + token.  Runs without gradients and without dropout."""
        missing = [n for n, v in (("input_ids", input_ids), ("encoder_input_ids", encoder_input_ids)) if v is None]
        if missing:
            raise _MissingArguments("Cobra.generate", missing)
        self._check_generate(input_ids, encoder_input_ids, n_candidates, temperature, "n_candidates")
        with torch.no_grad():
            return self._generate(input_ids, encoder_input_ids, n_candidates, temperature)

    def beam_fusion(self, input_ids: Optional[torch.Tensor] = None, encoder_input_ids: Optional[torch.Tensor] = None,
                    item_dense_vecs: Optional[torch.Tensor] = None, item_sem_ids: Optional[torch.Tensor] = None, n_candidates: int = 10,
                    n_beam: int = 50, temperature: float = 1.0, alpha: float = 0.5) -> BeamFusionOutput:
        """cobra.py:679-760 on native generate(n_beam): each beam's best catalog row (item_dense_vecs [N, d_model], re-normalised as
        the reference does) and its similarity come from one sweep of the catalog, without the [B, n_beam, N] similarity; then
        alpha softmax(scores) + (1 - alpha) (max_sim + 1) / 2 and its top n_candidates (equal fused scores: the lower beam first).
        Equal similarities: the lower catalog row.  -> item_ids [B, n_candidates], sem_ids [B, n_candidates, C] (item_sem_ids [N, C]
        gathered), scores."""
        missing = [n for n, v in (("input_ids", input_ids), ("encoder_input_ids", encoder_input_ids), ("item_dense_vecs", item_dense_vecs),
                                  ("item_sem_ids", item_sem_ids)) if v is None]
        if missing:
            raise _MissingArguments("Cobra.beam_fusion", missing)
        self._check_catalog("Cobra.beam_fusion", n_candidates, n_beam, item_dense_vecs, item_sem_ids)
        self._check_generate(input_ids, encoder_input_ids, n_beam, temperature, "n_beam")
        require_cuda(item_dense_vecs, item_sem_ids)
        with torch.no_grad():
            gen = self._generate(input_ids, encoder_input_ids, n_beam, temperature)
            return self._fuse(gen, item_dense_vecs, item_sem_ids, n_candidates, n_beam, alpha)

    def _check_catalog(self, fn, n_candidates, n_beam, item_dense_vecs, item_sem_ids):
        if not 1 <= n_candidates <= n_beam:
            raise ValueError(f"{fn}: n_candidates {n_candidates} must lie in 1 .. n_beam ({n_beam})")
        if item_dense_vecs.dim() != 2 or item_dense_vecs.shape[1] != self.d_model or item_dense_vecs.shape[0] < 1:
            raise ValueError(f"{fn}: item_dense_vecs must be [N >= 1, {self.d_model}], got {tuple(item_dense_vecs.shape)}")
        N = item_dense_vecs.shape[0]
        if tuple(item_sem_ids.shape) != (N, self.C):
            raise ValueError(f"{fn}: item_sem_ids must be [{N}, {self.C}], got {tuple(item_sem_ids.shape)}")

    def _fuse(self, gen, item_dense_vecs, item_sem_ids, n_candidates, n_beam, alpha) -> BeamFusionOutput:
        """BeamFusion's catalog sweep and tail on the n_beam beams of gen"""
        dev = gen.scores.device
        B, N = gen.scores.shape[0], item_dense_vecs.shape[0]
        table = torch.empty(N, self.d_model, dtype=torch.bfloat16, device=dev)
        for s in range(0, N, _CATALOG_CHUNK):                   # F.normalize(item_dense_vecs), bf16, a chunk of rows at a time
            chunk = item_dense_vecs[s:s + _CATALOG_CHUNK].to(device=dev, dtype=torch.float32).contiguous()
            table[s:s + _CATALOG_CHUNK] = Fn.cast_rows_bf16(Fn.l2norm_fwd(chunk)[0])
        best, item = Fn.cobra_dense_match(Fn.cast_rows_bf16(gen.dense_vecs.reshape(-1, self.d_model).contiguous()), table)
        max_sim, best_item = best.view(B, n_beam), item.view(B, n_beam)
        fused = alpha * torch.softmax(gen.scores, dim=-1) + (1 - alpha) * ((max_sim + 1) / 2)
        top, idx = torch.sort(fused, dim=-1, descending=True, stable=True)
        item_ids = best_item.gather(1, idx[:, :n_candidates])
        return BeamFusionOutput(item_ids=item_ids, sem_ids=item_sem_ids[item_ids], scores=top[:, :n_candidates].contiguous())

    def _check_generate(self, input_ids, encoder_input_ids, K, temperature, k_name):
        """the refusals of generate / beam_fusion, before any launch; the item checks read one flag to the host"""
        C = self.C
        if input_ids.dim() != 2 or input_ids.shape[1] % C or encoder_input_ids.dim() != 3 or \
                tuple(encoder_input_ids.shape[:2]) != (input_ids.shape[0], input_ids.shape[1] // C) or input_ids.shape[0] < 1:
            raise ValueError(f"Cobra: input_ids [B, T*C] and encoder_input_ids [B, T, L] expected, got {tuple(input_ids.shape)} and "
                             f"{tuple(encoder_input_ids.shape)}")
        self._check_beams(K, temperature, k_name)
        T = input_ids.shape[1] // C
        if T * (C + 1) + C - 1 >= self.max_len:
            raise ValueError(f"Cobra: {T} items leave no positions for the generated tokens: T*(C+1) + C - 1 = {T * (C + 1) + C - 1} must "
                             f"be below max_len {self.max_len}")
        real = (input_ids != self.pad_id).view(-1, T, C)[:, :, C - 1]
        flag = int(((~real.any(1)).any().long() + 2 * (real[:, 1:] & ~real[:, :-1]).any().long()).item())
        if flag & 1:
            raise ValueError("Cobra: a user has no item")
        if flag & 2:
            raise ValueError("Cobra: a real item follows a pad item; pad items must come after a user's real ones")

    def _check_beams(self, K, temperature, k_name):
        V = self.sparse_head[0].out_features
        if not 1 <= K <= min(V, _MAX_BEAMS) or K * V > _MAX_CANDIDATES:
            raise ValueError(f"Cobra: {k_name} {K} must lie in 1 .. min(id_vocab_size, {_MAX_BEAMS}) = {min(V, _MAX_BEAMS)} with "
                             f"{k_name} * id_vocab_size <= {_MAX_CANDIDATES}")
        if not temperature > 0:
            raise ValueError(f"Cobra: temperature must be positive, got {temperature}")

    def _generate(self, input_ids, encoder_input_ids, K, temperature) -> CobraGenerationOutput:
        require_cuda(input_ids, encoder_input_ids)
        ensure_device(input_ids.device)
        training = self.training
        self.train(False)                             # no dropout; restored below
        try:
            return self._beam_search(input_ids, encoder_input_ids, K, temperature)
        finally:
            self.train(training)

    def _beam_search(self, input_ids, encoder_input_ids, K, temperature):
        B, TC = input_ids.shape
        C = self.C
        T, L = TC // C, encoder_input_ids.shape[2]
        dev = input_ids.device
        # prefill: the histories once, each layer's QKV kept
        mask_items = (input_ids != self.pad_id).view(B, T, C)
        keep = mask_items[:, :, C - 1].reshape(-1).to(torch.uint8).contiguous()
        vecs = self._encode(encoder_input_ids.reshape(B * T, L), keep).view(B, T, -1)
        emb, seq_mask = self._interleave(input_ids, vecs, mask_items)
        hist_qkv = []
        h = self._decode(emb, seq_mask, hist_qkv)
        hist_len = (mask_items[:, :, C - 1].sum(1) * (C + 1)).to(torch.int32)
        h = h[torch.arange(B, device=dev), hist_len.long() - 1]                       # the last dense position: codebook 0

        def attend(i, q, suf, anc, S, H):
            return Fn.cobra_beam_attention(q, hist_qkv[i], hist_len, suf, anc, S, H)
        return self._beams(h, hist_len, K, temperature, attend)

    def _beams(self, h, hist_len, K, temperature, attend):
        """The beam search from each user's codebook-0 row h [B, D] (the final layer at the last dense position) over histories of
        hist_len [B] int32 decoder rows, whose K | V attend(layer, q, suffix QKV, ancestry, S, heads) reads."""
        e = self.cobra_emb
        B = h.shape[0]
        C, D = self.C, self.d_model
        dev = h.device
        head = self.sparse_head[0]
        tokens, scores, _, _ = Fn.cobra_beam_topk(_LinearF32Fn.apply(h, head.weight, head.bias).contiguous(), None, B, K, temperature)
        seqs = tokens.unsqueeze(-1)
        h_last = h.unsqueeze(1).expand(B, K, D) if C == 1 else None
        # extension: one new token per beam and codebook, attending to its user's history and its own earlier tokens
        layers = self.decoder.decoder.layers
        R = B * K
        suf = [torch.empty(C - 1, R, 3 * D, dtype=torch.bfloat16, device=dev) for _ in layers] if C > 1 else []
        w = [(Fn.cast_bf16(l.self_attn.in_proj_weight), Fn.cast_bf16(l.self_attn.out_proj.weight)) for l in layers] if C > 1 else []
        pos = hist_len.long().repeat_interleave(K)
        anc = None
        for c in range(1, C):
            tok = tokens.reshape(-1) + (c - 1) * e.id_vocab_size
            x = e.id_embed.weight[tok] + e.pos_embed.weight[pos + (c - 1)] + e.type_embed.weight[0]
            for i, layer in enumerate(layers):
                x = self._cached_layer(i, layer, x, w[i], lambda qkv: attend(i, qkv[:, :D], suf[i], anc, c, layer.self_attn.num_heads),
                                       suf[i][c - 1])
            head = self.sparse_head[c]
            logits = _LinearF32Fn.apply(x, head.weight, head.bias).contiguous()
            tokens, scores, parents, anc = Fn.cobra_beam_topk(logits, scores, B, K, temperature, anc)
            seqs = torch.cat([seqs.gather(1, parents.unsqueeze(-1).expand(-1, -1, c)), tokens.unsqueeze(-1)], dim=-1)
            if c == C - 1:
                h_last = x.view(B, K, D).gather(1, parents.unsqueeze(-1).expand(-1, -1, D))
        dense = Fn.l2norm_fwd(h_last.contiguous())[0]
        return CobraGenerationOutput(sem_ids=seqs, dense_vecs=dense, scores=scores)

    def _cached_layer(self, i, layer, x, w, attend, qkv=None):
        """decoder layer i on rows x [R, D] fp32 whose keys are cached: the QKV GEMM (into qkv when given), attend(qkv) -> the
        attention [R, D] bf16, the out-projection and _layer_tail; w = the bf16 (in_proj, out_proj) weights"""
        sa = layer.self_attn
        qkv, _ = Fn.linear_fwd(Fn.cast_rows_bf16(x.contiguous()), w[0], sa.in_proj_bias.detach().contiguous(), 0, out=qkv)
        A = attend(qkv)
        a, _ = Fn.linear_fwd(A, w[1], sa.out_proj.bias.detach().contiguous(), 0)
        return self._layer_tail(i, layer, x, a.float(), 0)

    # ---- serving from a paged pool
    def new_pool(self, max_users: int, num_pages: int, page_size: int = 64, max_items: Optional[int] = None) -> CobraPool:
        """A paged K | V pool for up to ``max_users`` users of at most ``max_items`` items each; ``page_size`` counts decoder
        positions, a positive multiple of 64.  The default and upper bound of ``max_items`` is the most items that leave generate its
        C - 1 positions below max_len and whose n (C+1) decoder rows fit the paged attention's 8192 history keys."""
        C = self.C
        limit = min((self.max_len - C) // (C + 1), _MAX_KEYS // (C + 1))
        max_items = limit if max_items is None else max_items
        if max_users < 1 or num_pages < 1:
            raise ValueError(f"Cobra.new_pool: max_users and num_pages must be positive, got {max_users}, {num_pages}")
        if page_size < 64 or page_size % 64:
            raise ValueError(f"Cobra.new_pool: page_size must be a positive multiple of 64 (one key tile), got {page_size}")
        if not 1 <= max_items <= limit:
            raise ValueError(f"Cobra.new_pool: max_items must lie in 1 .. {limit} (T (C+1) + C - 1 below max_len "
                             f"{self.max_len}, at most {_MAX_KEYS} decoder rows), got {max_items}")
        dev = self.cobra_emb.pos_embed.weight.device
        require_cuda(self.cobra_emb.pos_embed.weight)
        return CobraPool(max_users, num_pages, page_size, max_items, len(self.decoder.decoder.layers), self.d_model, C, dev)

    def _check_pool(self, pool: CobraPool):
        if not isinstance(pool, CobraPool) or pool.C != self.C or pool.kv.shape[0] != len(self.decoder.decoder.layers) or \
                pool.kv.shape[3] != 2 * self.d_model:
            raise ValueError("Cobra: the pool was not made by this model's new_pool")
        versions = tuple(p._version for p in self.parameters())
        if pool.param_versions is not None and pool.param_versions != versions:
            raise RuntimeError("genrec_b200: the model's parameters changed after this pool was written; rebuild the pool")
        return versions

    def extend_users(self, pool: CobraPool, users, input_ids: torch.Tensor, encoder_input_ids: torch.Tensor) -> None:
        """Append row b's real items to user ``users[b]``: input_ids [B, n C] with pad items after the real ones, encoder_input_ids
        [B, n, L] right-padded with 0 (generate's layout).  Only the new items' texts are encoded and only their n_b (C+1) decoder rows
        run through the layers, at the positions that continue the user's history; each layer writes their K | V into the user's pages
        and then attends from the pages.  An all-pad row leaves its user untouched.  Refusals (ValueError) come before any launch."""
        versions = self._check_pool(pool)
        C = self.C
        if input_ids.dim() != 2 or input_ids.shape[1] % C or input_ids.shape[1] == 0 or encoder_input_ids.dim() != 3 or \
                tuple(encoder_input_ids.shape[:2]) != (input_ids.shape[0], input_ids.shape[1] // C) or input_ids.shape[0] < 1:
            raise ValueError(f"Cobra.extend_users: input_ids [B, n*C] and encoder_input_ids [B, n, L] expected, got {tuple(input_ids.shape)} "
                             f"and {tuple(encoder_input_ids.shape)}")
        u = pool._users(users, "Cobra.extend_users")
        B, n = input_ids.shape[0], input_ids.shape[1] // C
        if len(u) != B:
            raise ValueError(f"Cobra.extend_users: {len(u)} users for {B} rows")
        # an item is real in all C codebooks or pad in all: the rows that run (every codebook's flag, _interleave) are then exactly
        # the n_b (C+1) rows the host lays out below from the last codebook's flags
        codes = (input_ids != self.pad_id).view(B, n, C)
        real = codes[:, :, C - 1]
        flags = torch.stack([(real[:, 1:] & ~real[:, :-1]).any(), (codes.any(-1) != codes.all(-1)).any()]).long()
        *counts, gap, partial = torch.cat([real.sum(1), flags]).tolist()                                        # one host read
        if partial:
            raise ValueError("Cobra.extend_users: an item has pad_id in some of its codebooks but not all; an item is real in all "
                             "C codebooks or pad in all")
        if gap:
            raise ValueError("Cobra.extend_users: a real item follows a pad item; pad items must come after a user's real ones")
        over = [x for x, k in zip(u, counts) if pool.lengths[x] + k > pool.max_items]
        if over:
            raise ValueError(f"Cobra.extend_users: users {over[:8]} would exceed max_items ({pool.max_items}); release them first")
        need = sum(pool._pages_for(pool.lengths[x] + k) - pool._pages_for(pool.lengths[x]) for x, k in zip(u, counts))
        if need > len(pool.free):
            raise ValueError(f"Cobra.extend_users: the call needs {need} pages and {len(pool.free)} are free; release users first")
        if not any(counts):
            return
        require_cuda(input_ids, encoder_input_ids)
        ensure_device(input_ids.device)
        training = self.training
        self.train(False)
        try:
            with torch.no_grad():
                self._extend(pool, u, counts, input_ids, encoder_input_ids, versions)
        finally:
            self.train(training)

    def _extend(self, pool, u, counts, input_ids, encoder_input_ids, versions):
        C, D = self.C, self.d_model
        B, n, L = encoder_input_ids.shape
        dev = input_ids.device
        mask_items = (input_ids != self.pad_id).view(B, n, C)
        keep = mask_items[:, :, C - 1].reshape(-1).to(torch.uint8).contiguous()
        vecs = self._encode(encoder_input_ids.reshape(B * n, L), keep).view(B, n, -1)   # refuses a malformed text before any write
        # the host bookkeeping: pages in row order, then one copy of the call's index arrays
        rows = [b for b in range(B) if counts[b]]
        start = [pool.lengths[u[b]] * (C + 1) for b in range(B)]
        for b in rows:
            x = u[b]
            for _ in range(pool._pages_for(pool.lengths[x] + counts[b]) - len(pool.pages[x])):
                pool.pages[x].append(pool.free.pop())
            pool.lengths[x] += counts[b]
        pool.param_versions = versions
        cols = pool.page_table.shape[1]
        table = torch.zeros(len(rows), cols, dtype=torch.int32)
        for i, b in enumerate(rows):
            table[i, :len(pool.pages[u[b]])] = torch.tensor(pool.pages[u[b]], dtype=torch.int32)
        new = [counts[b] * (C + 1) for b in rows]
        q_off = [0]
        for k in new:
            q_off.append(q_off[-1] + k)
        R = q_off[-1]
        users = [u[b] for b in rows]
        hist = [start[b] + k for b, k in zip(rows, new)]
        row_pos = [start[b] + j for b, k in zip(rows, new) for j in range(k)]
        row_user = [u[b] for b, k in zip(rows, new) for _ in range(k)]
        meta = torch.tensor(users + hist + q_off + row_pos + row_user + [p + 1 for p in row_pos], dtype=torch.int32).to(dev)
        nb = len(rows)
        users_d, hist_d, q_off_d = meta[:nb], meta[nb:2 * nb], meta[2 * nb:3 * nb + 1]
        pos_d, user_d, keys_d = meta[3 * nb + 1:3 * nb + 1 + R], meta[3 * nb + 1 + R:3 * nb + 1 + 2 * R], meta[3 * nb + 1 + 2 * R:]
        pool.page_table.index_copy_(0, users_d.long(), table.to(dev))
        # the new items' decoder rows, packed in row order, at positions that continue each history
        emb, seq_mask = self._interleave(input_ids, vecs, mask_items, torch.tensor(start, dtype=torch.int64).to(dev))
        x = emb[seq_mask]
        ps, max_keys = pool.page_size, max(hist)
        for i, layer in enumerate(self.decoder.decoder.layers):
            sa = layer.self_attn
            kv = pool.kv[i]

            def attend(qkv):
                Fn.cobra_kv_scatter(qkv, kv, pool.page_table, ps, user_d, pos_d)
                return Fn.cobra_paged_attention(qkv[:, :D], kv[..., :D], kv[..., D:], pool.page_table, ps, users_d, hist_d, max_keys, q_off_d,
                                                keys_d, sa.num_heads)
            x = self._cached_layer(i, layer, x, (Fn.cast_bf16(sa.in_proj_weight), Fn.cast_bf16(sa.out_proj.weight)), attend)
        pool.last_hidden.index_copy_(0, users_d.long(), x[q_off_d[1:].long() - 1])

    def _check_pool_users(self, pool, users, K, temperature, k_name, fn):
        self._check_pool(pool)
        u = pool._users(users, fn)
        self._check_beams(K, temperature, k_name)
        empty = [x for x in u if pool.lengths[x] == 0]
        if empty:
            raise ValueError(f"{fn}: users {empty[:8]} have no item")
        return u

    def _pool_beams(self, pool, u, K, temperature) -> CobraGenerationOutput:
        C, D = self.C, self.d_model
        dev = pool.kv.device
        ensure_device(dev)
        B = len(u)
        hist = [pool.lengths[x] * (C + 1) for x in u]
        meta = torch.tensor(u + hist + [b * K for b in range(B + 1)], dtype=torch.int32).to(dev)
        users_d, hist_d, q_off_d = meta[:B], meta[B:2 * B], meta[2 * B:]
        q_keys = hist_d.repeat_interleave(K)
        training = self.training
        self.train(False)

        def attend(i, q, suf, anc, S, H):
            kv = pool.kv[i]
            return Fn.cobra_paged_attention(q, kv[..., :D], kv[..., D:], pool.page_table, pool.page_size, users_d, hist_d, max(hist), q_off_d,
                                            q_keys, H, suf, anc, S)
        try:
            return self._beams(pool.last_hidden[users_d.long()], hist_d, K, temperature, attend)
        finally:
            self.train(training)

    def generate_users(self, pool: CobraPool, users, n_candidates: int = 10, temperature: float = 1.0) -> CobraGenerationOutput:
        """generate's beam search for each of ``users`` from the pool: started from the user's ``last_hidden``, generated token j at
        position n_u (C+1) + j, the history's K | V read from the user's pages.  Same outputs and order as generate."""
        u = self._check_pool_users(pool, users, n_candidates, temperature, "n_candidates", "Cobra.generate_users")
        with torch.no_grad():
            return self._pool_beams(pool, u, n_candidates, temperature)

    def beam_fusion_users(self, pool: CobraPool, users, item_dense_vecs: torch.Tensor, item_sem_ids: torch.Tensor, n_candidates: int = 10,
                          n_beam: int = 50, temperature: float = 1.0, alpha: float = 0.5) -> BeamFusionOutput:
        """beam_fusion on generate_users(n_beam): the same catalog sweep and fusion tail."""
        self._check_catalog("Cobra.beam_fusion_users", n_candidates, n_beam, item_dense_vecs, item_sem_ids)
        u = self._check_pool_users(pool, users, n_beam, temperature, "n_beam", "Cobra.beam_fusion_users")
        require_cuda(item_dense_vecs, item_sem_ids)
        with torch.no_grad():
            return self._fuse(self._pool_beams(pool, u, n_beam, temperature), item_dense_vecs, item_sem_ids, n_candidates, n_beam, alpha)
