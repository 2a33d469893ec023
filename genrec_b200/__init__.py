"""genrec_b200 - H100-native (sm_90a) implementation of the sequential-attention hot path of phonism/genrec.

Public surface (mirrors the reference's import paths through the thin ``genrec`` shim package at the repo root):
    genrec_b200.hstu    HSTU, HSTULayer, RelativePositionBias, TemporalBias
    genrec_b200.sasrec  SASRec, SASRecBlock, MultiHeadAttention, PointWiseFeedForward
    genrec_b200.rqvae   Quantize, RqVae (semantic-id path)
    genrec_b200.optim   FlatAdam (flat parameter / gradient / bf16-mirror buffers; one-pass reduce + Adam + broadcast over peer memory)
    genrec_b200.data    collate_jagged (device-side hstu / sasrec collate)
    genrec_b200.t5_attention   T5Attention (TIGER's attention module)
    genrec_b200.tiger_decode   TrieCSR, generate / beam_search (TIGER's trie-constrained beam search on the device)
    genrec_b200.ops     torch custom ops (genrec_b200::hstu_layer, hstu_attention, sasrec_attention, rq_residual_argmin, ...)
The compute runs in ``libgenrec_b200.so`` (C ABI in include/genrec_b200.h).  There is no CPU fallback.
"""
__version__ = "0.2.0"
