"""Plain-PyTorch autograd restatement of one PRM training step in the reference's own layout (position_transformer.py:98-186,
position_head.py:83-114, decoder.py:48-92, target_assign.py:32-53): Conv2d over (B, C, L, P) and a max over the points, the
memory encoder's 128-channel tap concatenated after the track's global max, torch's own multi_head_attention_forward with the
padding masks, the heads on (B, C, L), and the per-track loss loops.  Run on a copy of the module in float64 it is the reference
the device step is checked against; in float32 it measures what plain autograd of the same tree gets wrong (and how much memory
it keeps).  Dropout is applied as the module's configuration says; the tests set it to 0 where they compare.  The one deviation
kept from the device path: the heading bin of +pi is 11 (refine/modules.py TargetAssigner.encode_torch)."""
import copy

import numpy as np
import torch
import torch.nn.functional as F


def _mha(attn, q, k, mask, training):
    """(L, B, E) layout, key == value; need_weights so that torch runs the explicit bmm / softmax / dropout the reference's own
    MultiheadAttention runs (multi_head_attention.py:250-290), not a fused attention kernel"""
    return F.multi_head_attention_forward(q, k, k, attn.embed_dim, attn.num_heads, attn.in_proj_weight, attn.in_proj_bias, None, None,
                                          False, attn.dropout, attn.out_proj.weight, attn.out_proj.bias, training=training,
                                          key_padding_mask=mask, need_weights=True, average_attn_weights=False)[0]


def _decoder_layer(layer, query, key, query_pos, sa, ca, training):
    """decoder.py:48-92: query (B, E, L), key (B, E, N), query_pos (B, L, 4)"""
    qpe = layer.self_posembed.position_embedding_head(query_pos.transpose(1, 2)).permute(2, 0, 1)
    query, key = query.permute(2, 0, 1), key.permute(2, 0, 1)
    q = query + qpe
    query = layer.norm1(query + layer.dropout1(_mha(layer.self_attn, q, q, sa, training)))
    query = layer.norm2(query + layer.dropout2(_mha(layer.multihead_attn, query + qpe, key, ca, training)))
    query = layer.norm3(query + layer.dropout3(layer.linear2(layer.dropout(F.relu(layer.linear1(query))))))
    return query.permute(1, 2, 0)


def _heads(ffn, x):
    out = {}
    for head in ffn.heads:
        h = x
        for m in getattr(ffn, head):
            h = F.relu(m.bn(m.conv(h))) if hasattr(m, 'conv') else m(h)
        out[head] = h.permute(0, 2, 1)                                       # (B, L, C)
    return out


def targets(traj, gt, box_num):
    """target_assign.py:32-53, heading bin clamped to 0..11"""
    gt = gt.clone()
    h = gt[:, :, 6]
    h[h < -np.pi] += 2 * np.pi
    h[h > np.pi] -= 2 * np.pi
    anchors = (torch.arange(12, dtype=gt.dtype, device=gt.device) * (2 * np.pi / 12) - np.pi)[None, None]
    return {'center_reg': gt[:, :, :3] - traj[:, :, :3], 'heading_reg': (h.unsqueeze(-1) - anchors) / (np.pi / 12),
            'heading_cls': torch.floor((h + np.pi) / (np.pi / 6.)).long().clamp(0, 11), 'box_num': box_num}


def forward_loss(reg, batch, dtype=torch.float64):
    """the reference's forward and get_loss on ``reg`` (a PositionTransformer, used as it is) -> (loss, tb_dict)"""
    training = reg.training
    cast = lambda t: t.to(dtype)                                             # noqa: E731
    local, glob, traj = cast(batch['pos_query_points']), cast(batch['pos_memory_points']), cast(batch['pos_trajectory'])
    B, L, P, C = local.shape
    Pm = glob.shape[2]
    q = reg.query_encoder(local.permute(0, 3, 1, 2)).max(dim=3)[0]           # (B, E, L)
    q = reg.query_mlp(q)
    query_pos = torch.cat([traj[..., :3], traj[..., 6:]], dim=-1)
    g = glob.permute(0, 3, 1, 2).reshape(B, C, L * Pm)
    tap = reg.memory_encoder[:6](g)                                          # the forward hook on memory_encoder[5]
    m = reg.memory_encoder[6:](tap).max(dim=2, keepdim=True)[0]
    mem = reg.memory_mlp(torch.cat([m.repeat(1, 1, L * Pm), tap], dim=1))
    sa = batch['padding_mask'] != 0
    ca = sa.reshape(B, L, 1).repeat(1, 1, Pm).reshape(B, -1)
    dec = reg.decoder
    query = _decoder_layer(dec.decoder[0], q, mem, query_pos, sa, ca, training)
    preds = _heads(dec.prediction_heads[0], query)
    # the targets as the reference computes them, in the batch's own float32: in float64 the fold of a heading at float32 pi (which
    # is above pi) and a heading within rounding of a bin edge come out differently
    t = targets(batch['pos_trajectory'], batch['gt_pos_trajectory'], batch['box_num'])
    t['center_reg'], t['heading_reg'] = cast(t['center_reg']), cast(t['heading_reg'])
    bs = B
    cent = cls = dreg = 0
    for i in range(B):
        n = int(t['box_num'][i])
        cent = cent + (preds['center_reg'][i, :n] - t['center_reg'][i, :n]).abs().sum() / bs / n
        cls = cls + F.cross_entropy(preds['heading_cls'][i, :n], t['heading_cls'][i, :n]) / bs
        d = torch.gather((preds['heading_reg'][i, :n] - t['heading_reg'][i, :n]).abs(), 1, t['heading_cls'][i, :n].unsqueeze(-1))
        dreg = dreg + d.sum() / bs / n
    loss = cent + 0.1 * cls + 2 * dreg
    return loss, {'center_reg_loss': cent, 'heading_cls_loss': cls, 'heading_reg_loss': dreg, 'position_loss': loss}


def step(reg, batch, dtype=torch.float64):
    """one forward + backward on a copy of ``reg`` in ``dtype`` -> ({loss name: float}, {parameter name: gradient (dtype)})"""
    r = copy.deepcopy(reg).to(dtype)
    r.zero_grad(set_to_none=True)
    loss, tb = forward_loss(r, batch, dtype)
    loss.backward()
    return {k: float(v) for k, v in tb.items()}, {n: p.grad for n, p in r.named_parameters() if p.grad is not None}
