"""Float64 pure-PyTorch restatement of GeometryTransformer's train-mode forward and loss (geometry_transformer.py:75-194,
geometry_head.py:83-128, decoder.py:48-92, multi_head_attention.py:120-295, target_assign.py:17-29) on a state dict, with autograd
doing the backward -- TEST INFRASTRUCTURE.

Token-major: every 1x1 conv / Linear is a matmul on (rows, C), every BatchNorm takes batch statistics over all rows (F.batch_norm,
training), which is what BatchNorm1d over (B, C, L) computes.  BatchNorm statistics include padded points and queries, self-attention
does not mask padded queries; only the loss ignores them, as in the reference.  ``pooled_rows`` = {'memory': (B, 512), 'query':
(B*Q, 256)} rows within each group replaces each max-pool by a gather at those rows, so that a test can pool where the device did."""
import numpy as np
import torch
import torch.nn.functional as F

ANCHORS = ((4.8, 1.8, 1.5), (10.0, 2.6, 3.2), (2.0, 1.0, 1.6))
HEADS = 8


def grm_train_gt(seed, B, Q):
    """seeded ground-truth query boxes: sizes scattered around each of the three anchors"""
    g = np.random.default_rng([int(seed), 0x6E0])
    box = g.normal(0, 1, (B, Q, 7))
    anchor = np.asarray(ANCHORS)[g.integers(0, 3, (B, Q))]
    box[..., 3:6] = anchor * np.exp(g.normal(0, 0.25, (B, Q, 3)))
    return torch.from_numpy(box.astype(np.float32))


def grm_train_inputs(seed, B, **kw):
    """grm_inputs (geo_query_num of Q, then Q - 1) with seeded gt_geo_query_boxes"""
    from detzero_b200.synthetic import grm_inputs
    inp = grm_inputs(seed, B=B, **kw)
    inp['gt_geo_query_boxes'] = grm_train_gt(seed, B, inp['geo_query_boxes'].shape[1])
    return inp


class _Net:
    def __init__(self, sd, stats, dropout, generator, relu_masks=None):
        self.sd, self.stats, self.p, self.gen = sd, stats, dropout, generator
        self.masks = relu_masks or {}

    def conv(self, x, name):
        w = self.sd[name + '.weight']
        return F.linear(x, w.reshape(w.shape[0], -1), self.sd.get(name + '.bias'))

    def bn(self, x, name, eps, momentum):
        st = self.stats
        st[name + '.num_batches_tracked'] += 1
        return F.batch_norm(x, st[name + '.running_mean'], st[name + '.running_var'], self.sd[name + '.weight'], self.sd[name + '.bias'],
                            training=True, momentum=momentum, eps=eps)

    def cbr(self, x, conv, bn, eps=1e-3, momentum=0.01):
        h = self.bn(self.conv(x, conv), bn, eps, momentum)
        if bn in self.masks:                                  # the ReLU taken at a given mask: h where the mask is set, else 0
            return torch.where(self.masks[bn].to(h.device), h, torch.zeros_like(h))
        return torch.relu(h)

    def drop(self, x):
        return F.dropout(x, self.p, training=True) if self.p > 0 else x

    def ln(self, x, name):
        return F.layer_norm(x, x.shape[-1:], self.sd[name + '.weight'], self.sd[name + '.bias'], 1e-5)

    def mha(self, name, query, key, self_attention):
        B, Pq, E = query.shape
        Pk, hd = key.shape[1], E // HEADS
        W, b = self.sd[name + '.in_proj_weight'], self.sd[name + '.in_proj_bias']
        if self_attention:
            q, k, v = F.linear(query, W, b).chunk(3, dim=-1)
        else:
            q = F.linear(query, W[:E], b[:E])
            k, v = F.linear(key, W[E:], b[E:]).chunk(2, dim=-1)
        q = q * hd ** -0.5
        heads = lambda t, P: t.reshape(B, P, HEADS, hd).transpose(1, 2).reshape(B * HEADS, P, hd)    # noqa: E731
        w = self.drop(torch.softmax(torch.bmm(heads(q, Pq), heads(k, Pk).transpose(1, 2)), dim=-1))
        out = torch.bmm(w, heads(v, Pk)).view(B, HEADS, Pq, hd).transpose(1, 2).reshape(B, Pq, E)
        return self.conv(out, name + '.out_proj')


def _pool(y, groups, rows):
    y = y.view(groups, -1, y.shape[-1])
    if rows is None:
        return y.max(dim=1)[0]
    return y.gather(1, rows.long().to(y.device).unsqueeze(1)).squeeze(1)


def grm_train_step(state_dict, inputs, device='cpu', pooled_rows=None, dropout=0.0, generator=None, dtype=torch.float64, record=None,
                   relu_masks=None, path_outputs=None):
    """one training forward + backward in float64 (or ``dtype``).  state_dict: GeometryTransformer keys (no 'reg.' prefix); inputs: the data-dict
    keys geo_memory_points, geo_query_points, geo_query_boxes, geo_query_num, gt_geo_query_boxes.  Returns (losses {name: float},
    grads {param: tensor}, running stats after the step {buffer: tensor}).  ``record`` (a dict) receives the inputs of the two
    max-pools: 'memory' (B, N, 512) and 'query' (B*Q, P, 256), and the outputs of the two point paths: 'memory_out' (B*N, 256), the
    memory_mlp output, 'memory_pool' (B, 512) the pooled memory_encoder output, and 'query_pool' (B*Q, 256) the pooled
    query_encoder output.  ``relu_masks`` {BatchNorm name: bool (rows, C)} takes that layer's ReLU at the given mask instead of at
    the sign of its input, so that a test can restate a step at the masks the device took.  ``path_outputs`` {'memory_out',
    'query_pool'} replaces the two point paths' outputs by given tensors (constants: the point layers then get no gradient and are
    left out of grads), so that a test can restate the rest of the step from the device's point-path outputs"""
    stat_keys = ('running_mean', 'running_var', 'num_batches_tracked')
    sd = {k: v.to(device, dtype).clone().requires_grad_(True) for k, v in state_dict.items() if not k.endswith(stat_keys)}
    stats = {k: v.to(device).clone().to(dtype) if not k.endswith('num_batches_tracked') else v.to(device).clone()
             for k, v in state_dict.items() if k.endswith(stat_keys)}
    net = _Net(sd, stats, dropout, generator, relu_masks)
    pr = pooled_rows or {}
    m = inputs['geo_memory_points'].to(device, dtype)
    B, N, _ = m.shape
    x = m.reshape(B * N, -1)
    y1 = net.cbr(x, 'memory_encoder.0', 'memory_encoder.1')
    y2 = net.cbr(y1, 'memory_encoder.3', 'memory_encoder.4')                     # the hook on memory_encoder[5]
    y3 = net.cbr(y2, 'memory_encoder.6', 'memory_encoder.7')
    g = _pool(y3, B, pr.get('memory'))
    if record is not None:
        record['memory'] = y3.detach().view(B, N, -1)
        record['memory_pool'] = g.detach()
    x4 = torch.cat([y2.view(B, N, -1), g.unsqueeze(1).expand(B, N, g.shape[1])], dim=2).reshape(B * N, -1)
    mem = net.cbr(net.cbr(x4, 'memory_mlp.0', 'memory_mlp.1'), 'memory_mlp.3', 'memory_mlp.4')
    if record is not None:
        record['memory_out'] = mem.detach()
    if path_outputs is not None:
        mem = path_outputs['memory_out'].to(device, dtype)
    qp = inputs['geo_query_points'].to(device, dtype)
    _, Q, P, _ = qp.shape
    h = qp.reshape(B * Q * P, -1)
    for i in (0, 3, 6):
        h = net.cbr(h, 'query_encoder.%d' % i, 'query_encoder.%d' % (i + 1))
    q = _pool(h, B * Q, pr.get('query'))
    if record is not None:
        record['query'] = h.detach().view(B * Q, P, -1)
        record['query_pool'] = q.detach()
    if path_outputs is not None:
        q = path_outputs['query_pool'].to(device, dtype)
    q = net.cbr(net.cbr(q, 'query_mlp.0', 'query_mlp.1'), 'query_mlp.3', 'query_mlp.4')
    E = q.shape[1]
    query, key = q.view(B, Q, E), mem.view(B, N, E)
    d = 'decoder.decoder.0.'
    pe = d + 'self_posembed.position_embedding_head.'
    qpos = inputs['geo_query_boxes'][..., 3:6].to(device, dtype).reshape(B * Q, 3)
    qpe = net.conv(torch.relu(net.bn(net.conv(qpos, pe + '0'), pe + '1', 1e-5, 0.1)), pe + '3').view(B, Q, E)
    qin = query + qpe
    query = net.ln(query + net.drop(net.mha(d + 'self_attn', qin, qin, True)), d + 'norm1')
    query = net.ln(query + net.drop(net.mha(d + 'multihead_attn', query + qpe, key, False)), d + 'norm2')
    ff = net.conv(net.drop(torch.relu(net.conv(query, d + 'linear1'))), d + 'linear2')
    query = net.ln(query + net.drop(ff), d + 'norm3').reshape(B * Q, E)
    preds = {}
    for head in ('geometry_cls', 'geometry_reg'):
        hp = 'decoder.prediction_heads.0.%s.' % head
        hh = torch.relu(net.bn(net.conv(query, hp + '0.conv'), hp + '0.bn', 1e-5, 0.1))
        preds[head] = net.conv(hh, hp + '1').view(B, Q, -1)
    # targets (target_assign.py:17-29) and the loss over each track's first geo_query_num queries
    gt = inputs['gt_geo_query_boxes'].to(device, dtype)
    anchors = torch.tensor(ANCHORS, dtype=torch.float32).to(device, dtype)
    delta = (gt[..., 3:6].unsqueeze(2) - anchors) / anchors                        # (B, Q, 3 anchors, 3)
    cls_t = delta.abs().sum(-1).argmin(-1)
    num = [int(n) for n in inputs['geo_query_num']]
    cls_loss, reg_loss = 0, 0
    for b in range(B):
        n = num[b]
        cls_loss = cls_loss + F.cross_entropy(preds['geometry_cls'][b, :n], cls_t[b, :n])
        l1 = (preds['geometry_reg'][b, :n].view(n, 3, 3) - delta[b, :n]).abs()
        reg_loss = reg_loss + l1[torch.arange(n), cls_t[b, :n]].sum() / n
    cls_loss, reg_loss = cls_loss / B, reg_loss / B
    loss = 0.1 * cls_loss + 2 * reg_loss
    loss.backward()
    losses = {'cls_loss': cls_loss.item(), 'reg_loss': reg_loss.item(), 'geometry_loss': loss.item()}
    return losses, {k: v.grad.detach() for k, v in sd.items() if v.grad is not None}, stats


def probe(name, shape, seed):
    """the seeded tensor a gradient that is not stored in full is dotted with"""
    from detzero_b200.synthetic import seeded_tensor
    return seeded_tensor('probe.' + name, shape, seed).double()
