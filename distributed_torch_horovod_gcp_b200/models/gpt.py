"""Decoder-only transformer language model, GPT-2 small by default: 124 475 904 parameters in 148 tensors
(vocabulary 50 257 padded to 50 304, a multiple of 128, so the LM-head GEMM tiles evenly).

Token + learned position embedding, ``depth`` pre-LN blocks (``vit.EncoderBlock`` with ``causal=True``, so
attention runs on the causal flash-attention kernel, and LayerNorm eps 1e-5), a final LayerNorm, and an LM
head tied to the token embedding (``F2.linear(x, wte.weight)``, no bias).  Initialisation follows GPT-2:
N(0, 0.02) everywhere, with the residual projections (``proj``, ``fc2``) at 0.02 / sqrt(2 * depth).

``dropout`` (GPT-2 uses 0.1; default 0) is GPT-2's ``embd_pdrop``, ``attn_pdrop`` and ``resid_pdrop`` in one
value, as nanoGPT's ``dropout``: in training mode it drops the embedding sum, the attention probabilities and
the output of each residual branch.  Nothing is dropped inside the fused MLP node.

``sequence_parallel=True`` (world size > 1) splits each sequence across the ranks: ``forward`` takes this
rank's zigzag shard of the tokens (``ops.seq_parallel.zigzag_shard``), looks the position embedding up at the
shard's global positions, runs attention through ``sp_attention`` over every rank's keys and values, and
returns this rank's logits or the mean loss over its own tokens.  With equal shards, averaging the gradients
over the ranks (``DistributedOptimizer``) gives the full-sequence gradient.  At world size 1 the model is the
same as without it.

``sequence_parallel_size=G`` (G divides the world size) splits each sequence across a group of G ranks instead
of the whole world: the groups are the contiguous blocks of ranks [k G, (k + 1) G), a rank's sequence-parallel
rank is its index in its group, and each group trains on its own batch (sequence and data parallelism at once).
The constructor is then collective: for 1 < G < world it creates every group's ``hvd.ProcessSet``, in the same
order on every rank, or reuses a set already registered with the same ranks.  G = 1 is plain data parallelism and G = world the whole-world split.

The MLP is the fused node's exact (erf) GELU, not GPT-2's tanh approximation, so weights trained by the
original GPT-2 code would see a slightly different activation here.
"""
from __future__ import annotations

import math

from torch import nn

from ..ops import functional as F2
from ..ops import grad_sink
from .vit import EncoderBlock


class GPT(nn.Module):
    def __init__(self, vocab: int = 50304, context: int = 1024, depth: int = 12, heads: int = 12,
                 dim: int = 768, mlp_dim: int = 3072, dropout: float = 0.0, sequence_parallel: bool = False,
                 sequence_parallel_size=None):
        super().__init__()
        if not 0.0 <= dropout <= 1.0:
            raise ValueError(f"dropout must be in [0, 1], got {dropout}")
        if sequence_parallel and dropout > 0.0:
            raise ValueError("dropout is not supported with sequence_parallel=True")
        self.sequence_parallel = bool(sequence_parallel)
        self.sequence_parallel_size, self._sp_set = None, None
        if sequence_parallel_size is not None:
            self._sp_groups(int(sequence_parallel_size))
        self.vocab, self.context, self.dim = vocab, context, dim
        self.dropout = float(dropout)
        self.wte = nn.Embedding(vocab, dim)
        self.wpe = nn.Embedding(context, dim)
        self.layers = nn.ModuleList([EncoderBlock(dim, heads, mlp_dim, causal=True, eps=1e-5, dropout=dropout,
                                                  attention_dropout=dropout)
                                     for _ in range(depth)])
        self.ln_f = nn.LayerNorm(dim, eps=1e-5)
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, mean=0.0, std=0.02)
            if isinstance(m, nn.Linear):
                nn.init.zeros_(m.bias)
        for blk in self.layers:
            for lin in (blk.proj, blk.fc2):
                nn.init.normal_(lin.weight, mean=0.0, std=0.02 / math.sqrt(2 * depth))

    def forward(self, idx, targets=None):
        """``idx``: [B, S] int64 token ids, S <= context.  Without ``targets``: the logits [B * S, vocab] (rows
        in (b, s) order, ready for ``nn.CrossEntropyLoss`` against targets of shape [B * S]).  With ``targets``
        ([B, S] or [B * S]): the mean cross-entropy loss, through ``linear_cross_entropy`` on the LM head, which
        never materialises the logits on the kernel path.  Under sequence parallelism ``idx`` and ``targets`` are
        this rank's zigzag shards, and S the local length."""
        B, S = idx.shape
        rank, world = self._sp_rank_world()
        if S * world > self.context:
            raise ValueError(f"sequence length {S * world} exceeds the model's context of {self.context}")
        # the token embedding is also the LM head: two uses, so its gradient is summed by autograd
        # rather than written straight into the gradient bucket by the LM head's GEMM
        grad_sink.note_forward(self.wte.weight)
        if world > 1:
            from ..ops.seq_parallel import zigzag_positions
            x = self.wte(idx) + self.wpe.weight[zigzag_positions(S * world, rank, world, idx.device)]
        else:
            x = self.wte(idx) + self.wpe.weight[:S]
        if self.training and self.dropout > 0.0:
            x = F2.dropout_add(x, None, self.dropout)
        for blk in self.layers:
            x = blk(x, sequence_parallel=True, process_set=self._sp_set) if world > 1 else blk(x)
        x = F2.layer_norm(x, self.ln_f.weight, self.ln_f.bias, self.ln_f.eps)
        if targets is not None:
            return F2.linear_cross_entropy(x.reshape(B * S, self.dim), self.wte.weight, targets.reshape(-1))
        return F2.linear(x.reshape(B * S, self.dim), self.wte.weight)

    def _sp_groups(self, G: int):
        """Check ``sequence_parallel_size=G`` and take the process set of every group of G ranks (collective): a
        set registered with exactly those ranks is reused, so building several models does not add groups."""
        if not self.sequence_parallel:
            raise ValueError("sequence_parallel_size needs sequence_parallel=True")
        from .. import _state
        rt = _state.runtime()
        world = rt.size if rt.initialized else 1
        if G < 1 or world % G:
            raise ValueError(f"sequence_parallel_size must be a divisor of the world size {world}, got {G}")
        self.sequence_parallel_size = G
        if 1 < G < world:
            from ..torch.process_sets import add_process_set
            sets = []
            for k in range(world // G):
                ranks = list(range(k * G, (k + 1) * G))
                known = [ps for ps in rt.process_sets.values() if ps.ranks == ranks]
                sets.append(known[0] if known else add_process_set(ranks))
            self._sp_set = sets[rt.rank // G]

    def _sp_rank_world(self):
        """(rank, world) of the sequence split: (0, 1) unless ``sequence_parallel`` with world size > 1; with
        ``sequence_parallel_size=G``, the rank's index in its group of G contiguous ranks and G."""
        if not self.sequence_parallel:
            return 0, 1
        from .. import _state
        rt = _state.runtime()
        if not rt.initialized:
            return 0, 1
        G = self.sequence_parallel_size or rt.size
        return rt.rank % G, G


def gpt2(**kw):
    return GPT(**kw)


def gpt_tiny(**kw):
    """2 layers, 2 heads of 64 (the attention kernel's head dim), width 128, vocab 512, context 128."""
    d = dict(vocab=512, context=128, depth=2, heads=2, dim=128, mlp_dim=512)
    d.update(kw)
    return GPT(**d)
