"""Refiner (GRM / PRM / CRM) modules with the reference's names, constructor signatures and state-dict keys, running
token-major on libdetzero_b200:
  refining/detzero_refine/models/modules/transformer/multi_head_attention.py:7-295   MultiheadAttention
  refining/detzero_refine/models/modules/transformer/decoder.py:8-92                 TransformerDecoderLayer
  refining/detzero_refine/models/modules/transformer/position_encoding.py:4-21       PositionEmbeddingLearned
  refining/detzero_refine/models/modules/transformer/ffn.py:6-67                     FFN (prediction heads)
  refining/detzero_refine/models/modules/head/position_head.py, geometry_head.py     PositionHead / GeometryHead
  refining/detzero_refine/models/modules/{position,geometry}_transformer.py, confidence_pointnet.py
  refining/detzero_refine/models/modules/target_assign.py:73-104                     TargetAssigner.decode_torch
  utils/detzero_utils/model_utils.py:81-134                                          make_{linear,fc,conv}_layers

Layout: activations are (tokens, channels) row-major; the reference's (B,C,P) <-> (P,B,C) permute copies disappear.
Every 1x1 Conv / Linear (+BatchNorm eval +ReLU) is one fused GEMM launch; attention streams keys with an online
softmax and never materialises the (B*H, Pq, Pk) score tensor; the query scaling head_dim**-0.5 is folded into the
in-projection epilogue.  All three refiners also train (refine/train.py).
The ``forward_train`` methods follow the reference op for op through torch autograd, dropout included, token-major."""
import copy
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, ops
from . import train
from ..spconv.pytorch import fold_bn


def make_linear_layers(cfg, c_in, c_out, output_use_norm=False):
    layers = []
    for k in range(len(cfg)):
        layers += [nn.Linear(c_in, cfg[k], bias=False), nn.BatchNorm1d(cfg[k], eps=1e-3, momentum=0.01), nn.ReLU()]
        c_in = cfg[k]
    layers += [nn.Linear(c_in, c_out, bias=False), nn.BatchNorm1d(c_out, eps=1e-3, momentum=0.01), nn.ReLU()] \
        if output_use_norm else [nn.Linear(c_in, c_out, bias=True)]
    return nn.Sequential(*layers)


def make_fc_layers(cfg, c_in, c_out, output_use_norm=False):
    layers = []
    for k in range(len(cfg)):
        layers += [nn.Conv1d(c_in, cfg[k], kernel_size=1, bias=False), nn.BatchNorm1d(cfg[k], eps=1e-3, momentum=0.01), nn.ReLU()]
        c_in = cfg[k]
    layers += [nn.Conv1d(c_in, c_out, kernel_size=1, bias=False), nn.BatchNorm1d(c_out, eps=1e-3, momentum=0.01), nn.ReLU()] \
        if output_use_norm else [nn.Conv1d(c_in, c_out, kernel_size=1, bias=True)]
    return nn.Sequential(*layers)


def make_conv_layers(cfg, c_in, c_out, output_use_norm=False):
    layers = []
    for k in range(len(cfg)):
        layers += [nn.Conv2d(c_in, cfg[k], kernel_size=1, bias=False), nn.BatchNorm2d(cfg[k], eps=1e-3, momentum=0.01), nn.ReLU()]
        c_in = cfg[k]
    layers += [nn.Conv2d(c_in, c_out, kernel_size=1, bias=False), nn.BatchNorm2d(c_out, eps=1e-3, momentum=0.01), nn.ReLU()] \
        if output_use_norm else [nn.Conv2d(c_in, c_out, kernel_size=1, bias=True)]
    return nn.Sequential(*layers)


def _w2d(m, mode=_lib.DZ_F32, name='weight', rows=None):
    """weight of Linear / Conv1d(k=1) / Conv2d(k=1) (or the parameter `name` of m, rows [lo, hi) if given) as (N, K); rounded to
    TF32 (RN) once for the tensor-core mode: the tensor core truncates the fp32 container, and a weight it truncates biases every
    output toward zero.
    Cached on the module itself (not in a global keyed by id(): ids / addresses are recycled after a model is freed)."""
    w = getattr(m, name)
    ver = (w._version, w.data_ptr(), w.device)
    cache = m.__dict__.setdefault('_dz_w2d', {})
    key = (mode, name, rows)
    hit = cache.get(key)
    if hit is not None and hit[0] == ver:
        return hit[1]
    w2 = w.detach() if rows is None else w.detach()[rows[0]:rows[1]]
    w2 = w2.reshape(w2.shape[0], -1).contiguous().float()
    if mode == _lib.DZ_TF32:
        w2 = ops.round_tf32(w2)
    cache[key] = (ver, w2)
    return w2


def _first_group(mods, i=0):
    m = mods[i]
    assert isinstance(m, (nn.Linear, nn.Conv1d, nn.Conv2d)), type(m)
    bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], (nn.BatchNorm1d, nn.BatchNorm2d)) else None
    j = i + (2 if bn is not None else 1)
    relu = j < len(mods) and isinstance(mods[j], nn.ReLU)
    return m, bn, relu, j + (1 if relu else 0)


def _train_mlp(seq, x):
    """train-mode Conv1d(k=1) / BatchNorm1d / ReLU stack on token-major (rows, C) input through torch autograd: F.linear, not cuDNN
    Conv1d, so that it follows torch.backends.cuda.matmul.allow_tf32 (off by default) rather than cuDNN's TF32 default"""
    for m in seq:
        if isinstance(m, nn.Conv1d):
            x = F.linear(x, m.weight.squeeze(-1), m.bias)
        else:
            x = m(x)
    return x


def run_mlp_concat(seq, glob, per, gsize, mode, glob_first=True, pool=None):
    """``run_mlp(seq, cat([glob.expand over each group of gsize rows, per]))`` WITHOUT materialising the concatenation
    (position_transformer.py:118-123, geometry_transformer.py:131-136, confidence_pointnet.py:88-100 build it with expand + cat):
    the first layer's weight is split W = [W_g | W_p]; the global half is applied once per group (a tiny GEMM) and enters
    the per-row GEMM as a per-group shift (dz_linear_fwd_grouped).  glob (G, Cg), per (G*gsize, Cp)."""
    mods = list(seq.children())
    m, bn, relu, nxt = _first_group(mods)
    scale, shift = fold_bn(bn, m.bias) if bn is not None else (None, (None if m.bias is None else m.bias.detach().float()))
    Cg, Cp = glob.shape[1], per.shape[1]
    key = (mode, Cg, Cp, glob_first)
    cache = m.__dict__.setdefault('_dz_w2d_split', {})
    w = m.weight
    ver = (w._version, w.data_ptr(), w.device)
    hit = cache.get(key)
    if hit is None or hit[0] != ver:
        w32 = w.detach().reshape(w.shape[0], -1).float()
        assert w32.shape[1] == Cg + Cp
        wg, wp = (w32[:, :Cg], w32[:, Cg:]) if glob_first else (w32[:, Cp:], w32[:, :Cp])
        wg, wp = wg.contiguous(), wp.contiguous()
        if mode == _lib.DZ_TF32:
            wg, wp = ops.round_tf32(wg), ops.round_tf32(wp)
        hit = (ver, wg, wp)
        cache[key] = hit
    gshift = ops.linear(glob.contiguous(), hit[1], scale, None, False, mode=mode)                 # (G, N): (g W_g^T) * scale
    x = ops.linear_grouped(per.contiguous(), hit[2], gshift, gsize, scale, shift, relu, mode=mode)
    if pool and nxt >= len(mods):
        return ops.group_max(x, x.shape[0] // pool, pool)
    return run_mlp(seq, x, mode, start=nxt, pool=pool)


def run_mlp(seq, x, mode, upto=None, taps=None, start=0, pool=None):
    """token-major execution of a [Linear|Conv1x1] [BN] [ReLU] ... stack.  ``taps``: dict index -> output captured after
    module ``index`` (the reference's register_forward_hook on ``encoder[5]``).  ``pool = group``: the stack is followed by a max over
    groups of ``group`` consecutive rows (torch.max over a crop's points); in tensor-core mode the LAST layer and the pooling run as
    one kernel (dz_linear_max_fwd) and the (rows, C) activation is never written."""
    mods = list(seq.children())
    i = start
    while i < len(mods) and (upto is None or i < upto):
        m = mods[i]
        assert isinstance(m, (nn.Linear, nn.Conv1d, nn.Conv2d)), type(m)
        bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], (nn.BatchNorm1d, nn.BatchNorm2d)) else None
        j = i + (2 if bn is not None else 1)
        relu = j < len(mods) and isinstance(mods[j], nn.ReLU)
        if bn is not None:
            scale, shift = fold_bn(bn, m.bias)
        else:
            scale, shift = None, (None if m.bias is None else m.bias.detach().float())
        i = j + (1 if relu else 0)
        last = i >= len(mods) or (upto is not None and i >= upto)
        K = x.shape[1]
        if pool and last and mode == _lib.DZ_TF32 and pool % 128 == 0 and K % 32 == 0 and m.weight.shape[0] % 4 == 0 and x.shape[0] % pool == 0 \
                and not (taps is not None and (i - 1) in taps):
            return ops.linear_max(x, _w2d(m, mode), pool, scale, shift, relu, mode=mode)
        x = ops.linear(x, _w2d(m, mode), scale, shift, relu, mode=mode)
        if taps is not None and (i - 1) in taps:
            taps[i - 1] = x
    if pool:
        x = ops.group_max(x, x.shape[0] // pool, pool)
    return x


class PositionEmbeddingLearned(nn.Module):
    def __init__(self, input_channel, num_pos_feats=288):
        super().__init__()
        self.position_embedding_head = nn.Sequential(nn.Conv1d(input_channel, num_pos_feats, kernel_size=1),
                                                     nn.BatchNorm1d(num_pos_feats), nn.ReLU(inplace=True),
                                                     nn.Conv1d(num_pos_feats, num_pos_feats, kernel_size=1))

    def forward_tokens(self, xyz_tokens, mode):
        return run_mlp(self.position_embedding_head, xyz_tokens, mode)

    def forward_train(self, xyz_tokens):
        return _train_mlp(self.position_embedding_head, xyz_tokens)


class MultiheadAttention(nn.Module):
    """packed in-projection (3E,E) like the reference; forward_tokens works on (B, P, E) token-major tensors"""

    def __init__(self, embed_dim, num_heads, dropout=0., bias=True, add_bias_kv=False, add_zero_attn=False, kdim=None, vdim=None):
        super().__init__()
        assert not add_bias_kv and not add_zero_attn and kdim in (None, embed_dim) and vdim in (None, embed_dim)
        self.embed_dim, self.num_heads, self.dropout = embed_dim, num_heads, dropout
        self.head_dim = embed_dim // num_heads
        assert self.head_dim * num_heads == embed_dim
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * embed_dim)) if bias else None
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=bias)
        nn.init.xavier_uniform_(self.in_proj_weight)

    def _scaled(self, lo, hi, scale_q, mode):
        """(W[lo:hi], scale, shift) with the query scaling folded in for the first E rows (multi_head_attention.py:207)"""
        E = self.embed_dim
        w = _w2d(self, mode, 'in_proj_weight', (lo, hi))
        b = self.in_proj_bias.detach()[lo:hi].float() if self.in_proj_bias is not None else torch.zeros(hi - lo, device=w.device)
        s = torch.ones(hi - lo, device=w.device)
        if scale_q and lo == 0:
            s[:E] = float(self.head_dim) ** -0.5
        return w, s.contiguous(), (b * s).contiguous()

    def forward_tokens(self, query, key, key_padding_mask, mode, self_attention):
        """query (B,Pq,E); key == value (B,Pk,E) (the reference's qkv_same / kv_same branches, :129-157);
        key_padding_mask (B,Pk) uint8 or None.  Returns (B,Pq,E)."""
        B, Pq, E = query.shape
        Pk = key.shape[1]
        if self_attention:
            w, s, b = self._scaled(0, 3 * E, True, mode)
            qkv = ops.linear(query.reshape(B * Pq, E), w, s, b, False, mode=mode).view(B, Pq, 3 * E)
            q, k, v = qkv[:, :, :E], qkv[:, :, E:2 * E], qkv[:, :, 2 * E:]
        else:
            w, s, b = self._scaled(0, E, True, mode)
            q = ops.linear(query.reshape(B * Pq, E), w, s, b, False, mode=mode).view(B, Pq, E)
            w, s, b = self._scaled(E, 3 * E, False, mode)
            kv = ops.linear(key.reshape(B * Pk, E), w, None, b, False, mode=mode).view(B, Pk, 2 * E)
            k, v = kv[:, :, :E], kv[:, :, E:]
        att = ops.attention(q, k, v, key_padding_mask, self.num_heads, mode=mode)
        out = ops.linear(att.view(B * Pq, E), _w2d(self.out_proj, mode), None,
                         None if self.out_proj.bias is None else self.out_proj.bias.detach().float(), False, mode=mode)
        return out.view(B, Pq, E)

    def forward_train(self, query, key, self_attention, key_padding_mask=None):
        """multi_head_attention_forward (:120-295) through autograd: query (B,Pq,E), key == value (B,Pk,E) -> (B,Pq,E).
        key_padding_mask (B,Pk) bool or None: masked keys get -inf before the softmax, then dropout (:266-283)"""
        B, Pq, E = query.shape
        Pk, H = key.shape[1], self.num_heads
        W, b = self.in_proj_weight, self.in_proj_bias
        if self_attention:
            q, k, v = F.linear(query, W, b).chunk(3, dim=-1)
        else:
            q = F.linear(query, W[:E], None if b is None else b[:E])
            k, v = F.linear(key, W[E:], None if b is None else b[E:]).chunk(2, dim=-1)
        q = q * float(self.head_dim) ** -0.5
        heads = lambda t, P: t.reshape(B, P, H, self.head_dim).transpose(1, 2).reshape(B * H, P, self.head_dim)    # noqa: E731
        w = torch.bmm(heads(q, Pq), heads(k, Pk).transpose(1, 2))
        if key_padding_mask is not None:
            w = w.view(B, H, Pq, Pk).masked_fill(key_padding_mask.view(B, 1, 1, Pk), float('-inf')).view(B * H, Pq, Pk)
        w = F.softmax(w, dim=-1)
        w = F.dropout(w, p=self.dropout, training=self.training)
        out = torch.bmm(w, heads(v, Pk)).view(B, H, Pq, self.head_dim).transpose(1, 2).reshape(B, Pq, E)
        return F.linear(out, self.out_proj.weight, self.out_proj.bias)


class TransformerDecoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation='relu', self_posembed=None,
                 cross_posembed=None, cross_only=False):
        super().__init__()
        assert activation == 'relu'
        self.cross_only = cross_only
        if not self.cross_only:
            self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout)
        self.multihead_attn = MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(d_model), nn.LayerNorm(d_model), nn.LayerNorm(d_model)
        self.dropout1, self.dropout2, self.dropout3 = nn.Dropout(dropout), nn.Dropout(dropout), nn.Dropout(dropout)
        self.self_posembed = self_posembed
        self.cross_posembed = cross_posembed

    @staticmethod
    def _ln(norm, x, r):
        return ops.layernorm_residual(x, r, norm.weight.detach().float(), norm.bias.detach().float(), norm.eps)

    def forward_tokens(self, query, key, query_pos, key_pos, sa_mask, ca_mask, mode):
        """query (B,Pq,E), key (B,Pk,E) token-major; decoder.py:48-92 in eval mode (dropout = identity)"""
        B, Pq, E = query.shape
        qpe = None
        if self.self_posembed is not None:
            qpe = self.self_posembed.forward_tokens(query_pos.reshape(B * Pq, -1).contiguous(), mode).view(B, Pq, E)
        kpe = None
        if self.cross_posembed is not None and key_pos is not None:
            kpe = self.cross_posembed.forward_tokens(key_pos.reshape(-1, key_pos.shape[-1]).contiguous(), mode).view(B, -1, E)
        x = query.reshape(B * Pq, E)
        if not self.cross_only:
            qin = ops.add(query, qpe) if qpe is not None else query
            q2 = self.self_attn.forward_tokens(qin, qin, sa_mask, mode, True)
            x = self._ln(self.norm1, x, q2.reshape(B * Pq, E))
        qin = ops.add(x.view(B, Pq, E), qpe) if qpe is not None else x.view(B, Pq, E)
        kin = ops.add(key, kpe) if kpe is not None else key
        q2 = self.multihead_attn.forward_tokens(qin, kin, ca_mask, mode, False)
        x = self._ln(self.norm2, x, q2.reshape(B * Pq, E))
        h = ops.linear(x, _w2d(self.linear1, mode), None, self.linear1.bias.detach().float(), True, mode=mode)
        h = ops.linear(h, _w2d(self.linear2, mode), None, self.linear2.bias.detach().float(), False, mode=mode)
        x = self._ln(self.norm3, x, h)
        return x.view(B, Pq, E)

    def forward_train(self, query, key, query_pos, sa_mask=None, ca_mask=None):
        """decoder.py:48-92 in training (no key position embedding): query (B,Pq,E), key (B,Pk,E) -> (B,Pq,E); sa_mask (B,Pq) and
        ca_mask (B,Pk) bool key padding masks of the self- and cross-attention, or None"""
        B, Pq, E = query.shape
        qpe = None
        if self.self_posembed is not None:
            qpe = self.self_posembed.forward_train(query_pos.reshape(B * Pq, -1)).view(B, Pq, E)
        pos = (lambda t: t) if qpe is None else (lambda t: t + qpe)      # noqa: E731
        if not self.cross_only:
            q = pos(query)
            query = self.norm1(query + self.dropout1(self.self_attn.forward_train(q, q, True, sa_mask)))
        query = self.norm2(query + self.dropout2(self.multihead_attn.forward_train(pos(query), key, False, ca_mask)))
        h = self.linear2(self.dropout(F.relu(self.linear1(query))))
        return self.norm3(query + self.dropout3(h))


class ConvModule(nn.Module):
    """Conv1d(k=1, bias iff no norm) + BN1d + ReLU with the reference's attribute names (conv, bn)"""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.conv = nn.Conv1d(c_in, c_out, kernel_size=1, bias=False)
        self.bn = nn.BatchNorm1d(c_out)


class FFN(nn.Module):
    """prediction heads: per head Sequential(ConvModule(c,64), Conv1d(64, classes)) (ffn.py:21-50)"""

    def __init__(self, in_channels, heads, head_conv=64):
        super().__init__()
        self.heads = heads
        for head, (classes, num_conv) in heads.items():
            layers, c_in = [], in_channels
            for _ in range(num_conv - 1):
                layers.append(ConvModule(c_in, head_conv))
                c_in = head_conv
            layers.append(nn.Conv1d(head_conv, classes, kernel_size=1, bias=True))
            self.__setattr__(head, nn.Sequential(*layers))

    def forward_tokens(self, x, mode):
        out = {}
        for head in self.heads:
            h = x
            for m in getattr(self, head):
                if isinstance(m, ConvModule):
                    s, b = fold_bn(m.bn, None)
                    h = ops.linear(h, _w2d(m.conv, mode), s, b, True, mode=mode)
                else:
                    h = ops.linear(h, _w2d(m, mode), None, m.bias.detach().float(), False, mode=mode)
            out[head] = h
        return out

    def forward_train(self, x):
        """x (tokens, C): BatchNorm1d over the tokens takes the statistics of (B, C, Q)"""
        out = {}
        for head in self.heads:
            h = x
            for m in getattr(self, head):
                if isinstance(m, ConvModule):
                    h = F.relu(m.bn(F.linear(h, m.conv.weight.squeeze(-1))))
                else:
                    h = F.linear(h, m.weight.squeeze(-1), m.bias)
            out[head] = h
        return out


class _HeadBase(nn.Module):
    POS_DIMS = 4
    HEADS = {}

    def __init__(self, num_classes=3, num_decoder_layers=1, auxiliary=True, cross_only=False, memory_self_attn=False,
                 num_heads=8, hidden_channel=256, ffn_channel=256, dropout=0.1, bn_momentum=0.1, activation='relu',
                 bias='auto', **kwargs):
        super().__init__()
        self.num_classes, self.auxiliary, self.num_decoder_layers, self.bn_momentum = num_classes, auxiliary, num_decoder_layers, bn_momentum
        self.decoder = nn.ModuleList([
            TransformerDecoderLayer(hidden_channel, num_heads, ffn_channel, dropout, activation,
                                    self_posembed=PositionEmbeddingLearned(self.POS_DIMS, hidden_channel), cross_only=cross_only)
            for _ in range(num_decoder_layers)])
        self.prediction_heads = nn.ModuleList([FFN(hidden_channel, copy.deepcopy(self.heads_cfg(num_classes)))
                                               for _ in range(num_decoder_layers)])
        for m in self.decoder.parameters():
            if m.dim() > 1:
                nn.init.xavier_uniform_(m)
        for m in self.modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                m.momentum = self.bn_momentum


class PositionHead(_HeadBase):
    POS_DIMS = 4

    @staticmethod
    def heads_cfg(num_classes):
        return {'center_reg': (3, 2), 'heading_cls': (12, 2), 'heading_reg': (12, 2)}

    def forward_tokens(self, query, memory, query_pos, padding_mask, mode, mem_per_box):
        """position_head.py:83-114: sa mask = padding_mask, ca mask = padding_mask repeated per memory point"""
        B, L = padding_mask.shape
        sa = padding_mask.to(torch.uint8).contiguous()
        ca = sa.view(B, L, 1).expand(B, L, mem_per_box).reshape(B, -1).contiguous()
        rets = []
        for i in range(self.num_decoder_layers):
            query = self.decoder[i].forward_tokens(query, memory, query_pos, None, sa, ca, mode)
            rets.append(self.prediction_heads[i].forward_tokens(query.reshape(-1, query.shape[-1]), mode))
        return rets[-1] if self.auxiliary is False else rets[0]

    def forward_train(self, query, memory, query_pos, padding_mask, mem_per_box):
        """position_head.py:83-114 in training: the same masks as bool key padding masks, through autograd"""
        B, L = padding_mask.shape
        sa = padding_mask != 0
        ca = sa.view(B, L, 1).expand(B, L, mem_per_box).reshape(B, -1)
        rets = []
        for i in range(self.num_decoder_layers):
            query = self.decoder[i].forward_train(query, memory, query_pos, sa, ca)
            rets.append(self.prediction_heads[i].forward_train(query.reshape(-1, query.shape[-1])))
        return rets[-1] if self.auxiliary is False else rets[0]


class GeometryHead(_HeadBase):
    POS_DIMS = 3

    @staticmethod
    def heads_cfg(num_classes):
        return {'geometry_cls': (num_classes, 2), 'geometry_reg': (num_classes * 3, 2)}

    def forward_tokens(self, query, memory, query_pos, mode):
        rets = []
        for i in range(self.num_decoder_layers):
            query = self.decoder[i].forward_tokens(query, memory, query_pos, None, None, None, mode)
            rets.append(self.prediction_heads[i].forward_tokens(query.reshape(-1, query.shape[-1]), mode))
        if self.auxiliary is False:
            return {k: v.unsqueeze(0) for k, v in rets[-1].items()}
        return {k: torch.stack([r[k] for r in rets]) for k in rets[0]}          # (layers, B*Q, C)

    def forward_train(self, query, memory, query_pos):
        """geometry_head.py:83-128 in training: query (B,Q,E), memory (B,N,E) -> {head: (layers, B*Q, C)}"""
        rets = []
        for i in range(self.num_decoder_layers):
            query = self.decoder[i].forward_train(query, memory, query_pos)
            rets.append(self.prediction_heads[i].forward_train(query.reshape(-1, query.shape[-1])))
        if self.auxiliary is False:
            return {k: v.unsqueeze(0) for k, v in rets[-1].items()}
        return {k: torch.stack([r[k] for r in rets]) for k in rets[0]}


class TargetAssigner:
    """decode half of target_assign.py (:73-104) and its geometry- and confidence-mode encode (:17-29, :55-70)"""

    def __init__(self, anchor_sizes=None, mode='size', **kwargs):
        self.anchor_sizes = anchor_sizes
        self.anchor_slen = len(anchor_sizes) if anchor_sizes is not None else 0
        self.mode = mode
        self.dir_bin_num = 12
        self.anchor_angles = torch.arange(self.dir_bin_num, dtype=torch.float) * (2 * np.pi / self.dir_bin_num) - np.pi
        self.score_thresh = kwargs.get('score_thresh', [0.25, 0.5])

    def encode_torch(self, data_dict):
        """confidence mode: iou clamped to [0, 1]; negatives iou < th0, positives iou >= th1, the boxes between masked out.  A padded
        box (iou = -1) clamps to 0 and so enters the loss as a negative, as in the reference"""
        if self.mode == 'geometry':
            # size residuals against every anchor, (gt - anchor) / anchor; the class is the anchor with the least sum of |residual|
            gt = data_dict['gt_box']
            anchors = self.anchor_sizes.to(gt.device, gt.dtype).unsqueeze(0)
            delta = (gt[:, 3:6].unsqueeze(1) - anchors) / anchors
            return {'geometry_reg': delta.reshape(gt.shape[0], -1), 'geometry_cls': torch.min(delta.abs().sum(-1), dim=-1)[1]}
        if self.mode == 'position':
            # target_assign.py:32-53: gt heading folded into [-pi, pi], centre residual, heading residual against every bin's anchor
            # and the heading bin.  Deviation: floor((yaw + pi) / (pi / 6)) is 12 for yaw = pi and for float32 headings a few ulps
            # below it, a bin that does not exist (cross_entropy rejects it; on the device, a device-side assert).  +pi closes bin
            # 11, so 12 becomes 11.
            traj, gt = data_dict['pos_trajectory'], data_dict['gt_pos_trajectory']
            h = gt[..., 6]
            h = torch.where(h < -np.pi, h + 2 * np.pi, h)
            h = torch.where(h > np.pi, h - 2 * np.pi, h)
            anchors = self.anchor_angles.to(h.device, h.dtype)
            return {'center_reg': gt[..., :3] - traj[..., :3],
                    'heading_reg': (h.unsqueeze(-1) - anchors) / (np.pi / self.dir_bin_num),
                    'heading_cls': torch.floor((h + np.pi) / (np.pi / 6.)).long().clamp(0, self.dir_bin_num - 1),
                    'boxes_gt': torch.cat([gt[..., :6], h.unsqueeze(-1)], -1), 'box_num': data_dict['box_num']}
        if self.mode != 'confidence':
            raise NotImplementedError('TargetAssigner.encode_torch: mode %r' % (self.mode,))
        iou = torch.clamp(data_dict['iou'], 0, 1).reshape(-1)
        pos = iou >= self.score_thresh[1]
        return {'score_gt': pos.to(iou.dtype), 'iou_gt': iou, 'mask': (iou < self.score_thresh[0]) | pos}

    def decode_torch(self, preds, data_dict):
        if self.mode == 'geometry':
            reg = preds['geometry_reg']
            bs = reg.size(0)
            anchors = self.anchor_sizes.to(reg.device).unsqueeze(0).repeat(bs, 1, 1)
            reg = reg.reshape(bs, self.anchor_slen, 3) * anchors + anchors
            cls = torch.max(preds['geometry_cls'], dim=-1)[1].unsqueeze(-1).unsqueeze(-1).repeat(1, 1, 3)
            reg = torch.gather(reg, 1, cls).squeeze(1)
            return torch.cat([torch.zeros_like(reg), reg, torch.zeros_like(reg[:, 0:1])], dim=-1)
        bs, box_num, _ = preds['center_reg'].shape
        center = preds['center_reg'] + data_dict['pos_trajectory'][:, :, :3]
        angles = self.anchor_angles.to(center.device).view(1, 1, -1).repeat(bs, box_num, 1)
        dir_reg = preds['heading_reg'] * (np.pi / self.dir_bin_num) + angles
        dir_cls = torch.max(preds['heading_cls'], dim=-1)[1].unsqueeze(-1)
        return torch.cat([center, preds['size_reg'], torch.gather(dir_reg, 2, dir_cls)], dim=-1)


class PositionTransformer(nn.Module):
    """position_transformer.py:14-141"""

    def __init__(self, model_cfg, query_point_dims=None, memory_point_dims=None):
        super().__init__()
        self.model_cfg = model_cfg
        self.embed_dims = model_cfg.get('EMBED_DIMS', 256)
        self.mode = _lib.MODES[model_cfg.get('COMPUTE_MODE', 'fp32')]
        self.target_assigner = TargetAssigner(mode='position')
        self.query_encoder = make_conv_layers(model_cfg.QUERY_ENCODER, query_point_dims, self.embed_dims, True)
        self.query_mlp = make_fc_layers(model_cfg.REGRESSION_MLP, self.embed_dims, self.embed_dims, True)
        self.memory_encoder = make_fc_layers(model_cfg.MEMORY_ENCODER, memory_point_dims, self.embed_dims, True)
        self.memory_mlp = make_fc_layers(model_cfg.REGRESSION_MLP, self.embed_dims + model_cfg.MEMORY_ENCODER[1], self.embed_dims, True)
        dec = dict(model_cfg.DECODER)
        assert dec.pop('NAME') == 'PositionHead'
        self.decoder = PositionHead(**dec)
        self.preds_dict = {}
        self.targets_dict = {}
        self.loss_weight = [0.1, 2]
        self.pooled_rows = {}           # the rows the last training step's max-pools picked: 'memory' (B, 256), 'query' (B*L, 256);
        #                                 'memory_pool' (B, 256) the pooled memory_encoder output

    def forward(self, data_dict):
        if self.training:
            return self.forward_train(data_dict)
        return self.forward_eval(data_dict)

    def forward_train(self, data_dict):
        """position_transformer.py:98-139 in training: the query encoder and the memory path on the train-mode point layers
        (refine/train.py), the query MLP, position embedding, decoder and heads through autograd on this module's own layers,
        token-major, dropout included"""
        if self.mode == _lib.DZ_F32 and torch.backends.cuda.matmul.allow_tf32:
            raise RuntimeError('PositionTransformer with COMPUTE_MODE fp32 trains in fp32, but torch.backends.cuda.matmul.allow_tf32 is '
                               'set: the query MLP and the decoder would run TF32')
        local, glob, traj = data_dict['pos_query_points'].float(), data_dict['pos_memory_points'].float(), data_dict['pos_trajectory']
        B, L, P, C = local.shape
        Pm = glob.shape[2]
        if Pm != 48 or glob.shape[:2] != (B, L):
            raise ValueError('train-mode PositionTransformer needs pos_memory_points (B, L, 48, C) beside pos_query_points (B, L, P, C) '
                             '(position_head.py builds its cross-attention mask for 48 memory points per box); got %s and %s'
                             % (tuple(glob.shape), tuple(local.shape)))
        q = _train_mlp(self.query_mlp, train.prm_query(self, local))                    # (B*L, E)
        mem = train.prm_memory(self, glob)                                              # (B*L*Pm, E)
        E = q.shape[1]
        query_pos = torch.cat([traj[..., :3], traj[..., 6:]], dim=-1).float()
        preds = self.decoder.forward_train(q.view(B, L, E), mem.view(B, L * Pm, E), query_pos, data_dict['padding_mask'], Pm)
        preds = {k: v.view(B, L, -1) for k, v in preds.items()}
        preds['size_reg'] = traj[:, :, 3:6]
        self.preds_dict.update(preds)
        self.targets_dict.update(self.target_assigner.encode_torch(data_dict))
        return data_dict

    def get_loss(self, tb_dict=None):
        """position_transformer.py:143-186: per track over its first box_num boxes, the centre L1 summed / (bs * num), the heading
        cross entropy (mean) / bs and the L1 of the target bin's heading residual summed / (bs * num); center + 0.1 cls + 2 reg"""
        tb_dict = {} if tb_dict is None else tb_dict
        p, t = self.preds_dict, self.targets_dict
        B, L, _ = p['center_reg'].shape
        num = t['box_num'].to(p['center_reg'].device).long().clamp(1, L)
        valid = torch.arange(L, device=num.device).unsqueeze(0) < num.unsqueeze(1)                         # (B, L)
        cent = (p['center_reg'] - t['center_reg'].float()).abs().sum(-1)
        center_loss = (torch.where(valid, cent, 0).sum(1) / num).sum() / B
        ce = F.cross_entropy(p['heading_cls'].reshape(B * L, -1), t['heading_cls'].reshape(-1), reduction='none').view(B, L)
        cls_loss = (torch.where(valid, ce, 0).sum(1) / num).sum() / B
        reg = torch.gather((p['heading_reg'] - t['heading_reg'].float()).abs(), 2, t['heading_cls'].unsqueeze(-1)).squeeze(-1)
        reg_loss = (torch.where(valid, reg, 0).sum(1) / num).sum() / B
        tb_dict.update({'center_reg_loss': center_loss, 'heading_cls_loss': cls_loss, 'heading_reg_loss': reg_loss})
        w1, w2 = self.loss_weight
        loss = center_loss + w1 * cls_loss + w2 * reg_loss
        tb_dict['position_loss'] = loss
        return loss, tb_dict

    @torch.no_grad()
    def forward_eval(self, data_dict):
        local, glob, traj = data_dict['pos_query_points'], data_dict['pos_memory_points'], data_dict['pos_trajectory']
        B, L, P, C = local.shape
        Pm = glob.shape[2]
        mode = self.mode
        # query: per-point MLP -> max over the crop's points -> per-box MLP
        q = run_mlp(self.query_encoder, local.reshape(B * L * P, C).contiguous().float(), mode, pool=P)      # (B*L, E): MLP + max over the crop
        q = run_mlp(self.query_mlp, q, mode)                                             # (B*L, E)
        # memory: per-point MLP, global max over the track, concat [global, 128-ch intermediate] -> MLP
        taps = {5: None}
        g = run_mlp(self.memory_encoder, glob.reshape(B * L * Pm, C).contiguous().float(), mode, taps=taps, pool=L * Pm)     # (B, E)
        mem = run_mlp_concat(self.memory_mlp, g, taps[5], L * Pm, mode, glob_first=True)  # Linear(cat([global, 128-ch tap])) fused: (B*L*Pm, E)
        E = mem.shape[1]
        query_pos = torch.cat([traj[..., :3], traj[..., 6:]], dim=-1).float()
        data_dict['query'] = q.view(B, L, E).permute(0, 2, 1)                            # reference-shaped views (B,E,L)
        data_dict['memory'] = mem.view(B, L * Pm, E).permute(0, 2, 1)
        data_dict['query_pos'] = query_pos
        preds = self.decoder.forward_tokens(q.view(B, L, E), mem.view(B, L * Pm, E), query_pos, data_dict['padding_mask'] != 0,
                                            mode, Pm)
        preds = {k: v.view(B, L, -1) for k, v in preds.items()}
        preds['size_reg'] = traj[:, :, 3:6]
        self.preds_dict.update(preds)
        boxes = self.target_assigner.decode_torch(preds, data_dict)
        data_dict['batch_box_preds'] = boxes
        preds['batch_box_preds'] = boxes
        return data_dict


class GeometryTransformer(nn.Module):
    """geometry_transformer.py:11-156 (note the reference's swapped names: memory_encoder takes QUERY_POINT_DIMS)"""

    def __init__(self, model_cfg, query_point_dims=None, memory_point_dims=None):
        super().__init__()
        self.model_cfg = model_cfg
        self.embed_dims = model_cfg.get('EMBED_DIMS', 256)
        self.mode = _lib.MODES[model_cfg.get('COMPUTE_MODE', 'fp32')]
        self.anchor_sizes = model_cfg.get('ANCHOR_SIZES', [[4.8, 1.8, 1.5], [10.0, 2.6, 3.2], [2.0, 1.0, 1.6]])
        self.target_assigner = TargetAssigner(anchor_sizes=torch.tensor(self.anchor_sizes, dtype=torch.float), mode='geometry')
        E = self.embed_dims
        self.memory_encoder = make_fc_layers(model_cfg.MEMORY_ENCODER, query_point_dims, E * 2, True)
        self.memory_mlp = make_fc_layers(model_cfg.REGRESSION_MLP, E * 2 + model_cfg.MEMORY_ENCODER[1], E, True)
        self.query_encoder = make_fc_layers(model_cfg.QUERY_ENCODER, memory_point_dims, E, True)
        self.query_mlp = make_linear_layers(model_cfg.REGRESSION_MLP, E, E, True)
        dec = dict(model_cfg.DECODER)
        assert dec.pop('NAME') == 'GeometryHead'
        self.decoder = GeometryHead(**dec)
        self.preds_dict = {}
        self.targets_dict = {}
        self.loss_weight = [0.1, 2]
        self.pooled_rows = {}           # the rows the last training step's max-pools picked: 'memory' (B, 512), 'query' (B*Q, 256);
        #                                 'memory_pool' (B, 512) the pooled memory_encoder output

    def forward(self, data_dict):
        if self.training:
            return self.forward_train(data_dict)
        return self.forward_eval(data_dict)

    def forward_train(self, data_dict):
        """geometry_transformer.py:118-156 in training: the memory path and the query encoder on the device (refine/train.py), the
        query MLP, decoder and heads through autograd on this module's own layers, token-major"""
        if self.mode == _lib.DZ_F32 and torch.backends.cuda.matmul.allow_tf32:
            raise RuntimeError('GeometryTransformer with COMPUTE_MODE fp32 trains in fp32, but torch.backends.cuda.matmul.allow_tf32 is '
                               'set: the query MLP and the decoder would run TF32')
        mpts = data_dict['geo_memory_points'].float()
        B, N, _ = mpts.shape
        mem = train.grm_memory(self, mpts)                                              # (B*N, E)
        qpts = data_dict['geo_query_points'].float()
        Q = qpts.shape[1]
        q = _train_mlp(self.query_mlp, train.grm_query(self, qpts))                     # (B*Q, E)
        E = q.shape[1]
        qpos = data_dict['geo_query_boxes'][..., 3:6].float()
        preds = self.decoder.forward_train(q.view(B, Q, E), mem.view(B, N, E), qpos)
        preds = {k: v.view(v.shape[0], B, Q, -1) for k, v in preds.items()}               # (layers, B, Q, C)
        preds['geo_query_num'] = data_dict['geo_query_num']
        self.preds_dict.update(preds)
        self.targets_dict.update(self.assign_targets(data_dict))
        return data_dict

    def assign_targets(self, data_dict):
        """geometry_transformer.py:75-90: per query, (B, Q, 3 * anchors) residuals and (B, Q) classes"""
        gt = data_dict['gt_geo_query_boxes'].float()
        B, Q, _ = gt.shape
        t = self.target_assigner.encode_torch({'gt_box': gt.reshape(B * Q, -1)})
        return {'geometry_cls': t['geometry_cls'].view(B, Q), 'geometry_reg': t['geometry_reg'].view(B, Q, -1)}

    def get_loss(self, tb_dict=None):
        """geometry_transformer.py:158-194: per layer and track, over its first geo_query_num queries only, the mean cross entropy
        and the L1 of the target class's 3 residuals summed / query_num; each summed over tracks / B; 0.1 cls + 2 reg"""
        tb_dict = {} if tb_dict is None else tb_dict
        cls_p, reg_p = self.preds_dict['geometry_cls'], self.preds_dict['geometry_reg']
        layers, B, Q, C = cls_p.shape
        cls_t, reg_t = self.targets_dict['geometry_cls'], self.targets_dict['geometry_reg']
        num = self.preds_dict['geo_query_num'].to(cls_p.device).long()
        valid = torch.arange(Q, device=cls_p.device).unsqueeze(0) < num.unsqueeze(1)                        # (B, Q)
        cls_loss, reg_loss = 0, 0
        for li in range(layers):
            ce = F.cross_entropy(cls_p[li].reshape(B * Q, C), cls_t.reshape(-1), reduction='none').view(B, Q)
            cls_loss = cls_loss + (torch.where(valid, ce, 0).sum(1) / num).sum()
            l1 = (reg_p[li] - reg_t).abs().view(B, Q, -1, 3)
            l1 = torch.gather(l1, 2, cls_t.view(B, Q, 1, 1).expand(B, Q, 1, 3)).view(B, Q, 3)
            reg_loss = reg_loss + (torch.where(valid, l1.sum(-1), 0).sum(1) / num).sum()
        cls_loss, reg_loss = cls_loss / B, reg_loss / B
        tb_dict.update({'reg_loss': reg_loss, 'cls_loss': cls_loss})
        w1, w2 = self.loss_weight
        loss = w1 * cls_loss + w2 * reg_loss
        tb_dict['geometry_loss'] = loss
        return loss, tb_dict

    @torch.no_grad()
    def forward_eval(self, data_dict):
        mpts = data_dict['geo_memory_points'].float()
        B, N, C = mpts.shape
        mode = self.mode
        taps = {5: None}
        g = run_mlp(self.memory_encoder, mpts.reshape(B * N, C).contiguous(), mode, taps=taps, pool=N)
        mem = run_mlp_concat(self.memory_mlp, g, taps[5], N, mode, glob_first=False)                     # cat order: [intermediate, global]
        qpts = data_dict['geo_query_points'].float()
        _, Q, P, Cq = qpts.shape
        q = run_mlp(self.query_encoder, qpts.reshape(B * Q * P, Cq).contiguous(), mode, pool=P)
        q = run_mlp(self.query_mlp, q, mode)
        E = q.shape[1]
        qpos = data_dict['geo_query_boxes'][..., 3:6].float().contiguous()
        preds = self.decoder.forward_tokens(q.view(B, Q, E), mem.view(B, N, E), qpos, mode)
        preds = {k: v.view(v.shape[0], B, Q, -1) for k, v in preds.items()}               # (layers, B, Q, C)
        preds['geo_query_num'] = data_dict['geo_query_num']
        self.preds_dict.update(preds)
        data_dict['batch_box_preds'] = self.generate_predicted_boxes(preds, data_dict)
        return data_dict

    def generate_predicted_boxes(self, preds, data_dict):
        """geometry_transformer.py:91-116: per-query decode, mean over the valid queries, mean over layers"""
        layers, bs, qn, _ = preds['geometry_cls'].shape
        num = preds['geo_query_num']
        layer_boxes = []
        for li in range(layers):
            qb = torch.stack([self.target_assigner.decode_torch({'geometry_cls': preds['geometry_cls'][li][:, i],
                                                                 'geometry_reg': preds['geometry_reg'][li][:, i]}, data_dict)
                              for i in range(qn)], dim=1)
            layer_boxes.append(torch.stack([qb[b, :int(num[b])].mean(dim=0) for b in range(bs)], dim=0))
        return torch.stack(layer_boxes, dim=0).mean(0)


class ConfidencePointnet(nn.Module):
    """confidence_pointnet.py:9-113"""

    def __init__(self, model_cfg, query_point_dims=None, memory_point_dims=None):
        super().__init__()
        self.model_cfg = model_cfg
        E = self.embed_dims = model_cfg.get('EMBED_DIMS', 256)
        self.mode = _lib.MODES[model_cfg.get('COMPUTE_MODE', 'fp32')]
        self.pts_encoder_1 = make_conv_layers(model_cfg.ENCODER_MLP, query_point_dims, E, True)
        self.pts_encoder_2 = make_conv_layers([], E + model_cfg.ENCODER_MLP[1], E, True)
        self.pts_mlp = make_fc_layers(model_cfg.REGRESSION_MLP, E, E, True)
        self.regression_mlp = make_fc_layers(model_cfg.REGRESSION_MLP, E * 2, E, True)
        self.heads = nn.ModuleDict({t: make_fc_layers([int(E / 2)], E, 1, False) for t in ('score_reg', 'iou_reg')})
        self.preds_dict = {}
        self.targets_dict = {}
        self.score_thresh = model_cfg.get('SCORE_THRESH', [0.25, 0.5])
        self.loss_weight = [1.0, 1.0]
        self.target_assigner = TargetAssigner(mode='confidence', score_thresh=self.score_thresh)
        self.pooled_rows = {}           # the rows the last training step's max-pools picked: 'enc1', 'enc2' (B*L, 256)

    def forward(self, data_dict):
        if self.training:
            return self.forward_train(data_dict)
        return self.forward_eval(data_dict)

    def forward_train(self, data_dict):
        """confidence_pointnet.py:80-108 in training: the point encoders on the device (refine/train.py), the per-box part through
        autograd on this module's own layers, token-major ((B*L, C) rows: BatchNorm1d takes the same statistics as on (B, C, L))"""
        if self.mode == _lib.DZ_F32 and torch.backends.cuda.matmul.allow_tf32:
            raise RuntimeError('ConfidencePointnet with COMPUTE_MODE fp32 trains in fp32, but torch.backends.cuda.matmul.allow_tf32 is '
                               'set: the per-box layers would run TF32')
        pts = data_dict['conf_points'].float()
        B, L, P, C = pts.shape
        E = self.embed_dims
        pool = train.point_encoders(self, pts)                                          # (B*L, E)
        tap = _train_mlp(self.pts_mlp, pool)                                            # pts_mlp[5] == the stack's output
        gg = tap.view(B, L, E).max(dim=1)[0]
        out = _train_mlp(self.regression_mlp, torch.cat([gg.unsqueeze(1).expand(B, L, E), tap.view(B, L, E)], dim=2).reshape(B * L, 2 * E))
        preds = {t: torch.sigmoid(_train_mlp(self.heads[t], out).view(B, L, 1)) for t in ('score_reg', 'iou_reg')}
        self.preds_dict.update(preds)
        self.targets_dict.update(self.target_assigner.encode_torch(data_dict))
        return data_dict

    def get_loss(self, tb_dict=None):
        """confidence_pointnet.py:115-150: BCE (log clamped at -100) summed over the mask / the mask count, score and iou heads"""
        tb_dict = {} if tb_dict is None else tb_dict
        mask = self.targets_dict['mask']
        n = mask.sum()
        bin_cls_loss = F.binary_cross_entropy(self.preds_dict['score_reg'].reshape(-1)[mask], self.targets_dict['score_gt'][mask],
                                              reduction='none').sum() / n
        iou_loss = F.binary_cross_entropy(self.preds_dict['iou_reg'].reshape(-1)[mask], self.targets_dict['iou_gt'][mask],
                                          reduction='none').sum() / n
        w1, w2 = self.loss_weight
        conf_loss = bin_cls_loss * w1 + iou_loss * w2
        tb_dict.update({'bin_cls_loss': bin_cls_loss, 'iou_loss': iou_loss})
        tb_dict['confidence_loss'] = conf_loss
        return conf_loss, tb_dict

    @torch.no_grad()
    def forward_eval(self, data_dict):
        pts = data_dict['conf_points'].float()
        B, L, P, C = pts.shape
        mode = self.mode
        taps = {5: None}
        g = run_mlp(self.pts_encoder_1, pts.reshape(B * L * P, C).contiguous(), mode, taps=taps, pool=P)    # (B*L, E)
        pool = run_mlp_concat(self.pts_encoder_2, g, taps[5], P, mode, glob_first=True, pool=P)
        taps2 = {5: None}
        pool = run_mlp(self.pts_mlp, pool, mode, taps=taps2)                             # (B*L, E); tap = after pts_mlp[5]
        gg = ops.group_max(pool, B, L)                                                   # (B, E)
        out = run_mlp_concat(self.regression_mlp, gg, taps2[5], L, mode, glob_first=True)
        preds = {t: torch.sigmoid(run_mlp(self.heads[t], out, mode).view(B, L, 1)) for t in ('score_reg', 'iou_reg')}
        self.preds_dict.update(preds)
        data_dict['pred_score'] = torch.sqrt(preds['score_reg'].squeeze(2) * preds['iou_reg'].squeeze(2))
        return data_dict


#: registry, same keys as refining/detzero_refine/models/refine_template.py:11-15
refine_modules = {'GeometryTransformer': GeometryTransformer, 'PositionTransformer': PositionTransformer,
                  'ConfidencePointnet': ConfidencePointnet}


class RefineTemplate(nn.Module):
    """refine_template.py:18-77: builds ``self.reg`` by NAME from the config"""

    def __init__(self, model_cfg, dataset=None):
        super().__init__()
        self.model_cfg = model_cfg
        self.dataset = dataset
        self.tta = getattr(dataset, 'tta', False)
        self.register_buffer('global_step', torch.LongTensor(1).zero_())
        self.add_module('reg', refine_modules[model_cfg.REGRESSION['NAME']](
            model_cfg=model_cfg.REGRESSION, query_point_dims=model_cfg.get('QUERY_POINT_DIMS', 0),
            memory_point_dims=model_cfg.get('MEMORY_POINT_DIMS', 0)))

    def update_global_step(self):
        self.global_step += 1

    def get_training_loss(self):
        """refine_template.py:52-62"""
        disp_dict = {}
        loss, tb_dict = self.reg.get_loss({})
        tb_dict['full_loss'] = loss
        return loss, tb_dict, disp_dict

    def forward(self, data_dict):
        data_dict = self.reg(data_dict)
        if self.training:
            loss, tb_dict, disp_dict = self.get_training_loss()
            return {'loss': loss}, tb_dict, disp_dict
        key = 'pred_score' if 'pred_score' in data_dict else 'batch_box_preds'
        return {('pred_score' if key == 'pred_score' else 'pred_boxes'): data_dict[key]}, {}, {}


refine_models = {'GeometryRefineModel': RefineTemplate, 'PositionRefineModel': RefineTemplate, 'ConfidenceRefineModel': RefineTemplate}


def build_network(model_cfg, dataset=None):
    return refine_models[model_cfg.NAME](model_cfg=model_cfg, dataset=dataset)
