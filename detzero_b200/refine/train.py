"""Train-mode CRM point encoders: ``pts_encoder_1 -> max over the crop's points -> pts_encoder_2 -> max over points``
(confidence_pointnet.py:85-92) as one autograd Function on libdetzero_b200 (csrc/refine_train.cu).

The reference keeps, per point row, every layer's conv and ReLU output and the 384-channel concatenation for autograd (about
1 950 floats per row).  Here the saved state is the input points, per layer the batch mean and variance, and per (crop, channel)
the pooled row and its pre-activation; the point layers are recomputed tile by tile in each pass.

BatchNorm2d takes its statistics over all B*L*P rows (padded boxes included), normalises with the biased variance and updates
``running_var`` with the unbiased one, as torch does.  The gradient of a max goes to one maximal row, the lowest on ties; a ReLU
output of 0 passes no gradient (threshold_backward).  Ties at a positive value only arise between identical rows, which give
identical weight gradients, so the choice changes no parameter gradient."""
import torch

from .. import _lib, ops

C1, C2, C3, C4 = 128, 128, 256, 256


def _bn_update(bn, mean, var, n):
    with torch.no_grad():
        m = bn.momentum
        bn.running_mean.mul_(1 - m).add_(mean.float(), alpha=m)
        bn.running_var.mul_(1 - m).add_((var * (n / max(n - 1, 1))).float(), alpha=m)
        bn.num_batches_tracked.add_(1)


class CrmPointEncoders(torch.autograd.Function):
    """x (crops*P, c0) -> (crops, 256).  ``rows`` (a dict) receives the pooled row of each (crop, channel) under 'enc1' and 'enc2'.
    Arguments after ``bns`` (the four BatchNorm2d modules, whose running statistics the forward updates): per layer the conv weight,
    BN weight and BN bias."""

    @staticmethod
    def forward(ctx, x, P, mode, rows, bns, w1, g1, b1, w2, g2, b2, w3, g3, b3, w4, g4, b4):
        R, c0 = x.shape
        crops, dev = R // P, x.device
        W1, W2, W3, W4 = (w.detach().reshape(w.shape[0], -1).float() for w in (w1, w2, w3, w4))
        if (W1.shape[0], W2.shape, W3.shape, W4.shape) != (C1, (C2, C1), (C3, C2), (C4, C3 + C2)):
            raise ValueError('train-mode ConfidencePointnet supports ENCODER_MLP [128, 128] and EMBED_DIMS 256; got layer weights %s'
                             % [tuple(w.shape) for w in (W1, W2, W3, W4)])
        W4g, W4p = W4[:, :C3].contiguous(), W4[:, C3:].contiguous()
        wf = (W1.t().contiguous(), W2.t().contiguous(), W3.t().contiguous(), W4p.t().contiguous())
        wb = (W2.contiguous(), W3.contiguous(), W4p)
        tab = torch.zeros(4, 6, 256, dtype=torch.float32, device=dev)
        stats = torch.empty(512, dtype=torch.float64, device=dev)
        zext = torch.empty(2, crops, 256, dtype=torch.float32, device=dev)
        iext = torch.empty(2, crops, 256, dtype=torch.int32, device=dev)
        csum = torch.empty(crops, 256, dtype=torch.float64, device=dev)
        shift4 = None
        per, sels, zsels = [], [], []
        for l, (C, gam, bet, bn) in enumerate(zip((C1, C2, C3, C4), (g1, g2, g3, g4), (b1, b2, b3, b4), bns), 1):
            ops.crm_point_pass(l, mode, x, P, wf, wb, tab, shift4, zext=zext, iext=iext, csum=csum, stats=stats)
            mean = stats[:C] / R
            var = (stats[256:256 + C] / R - mean * mean).clamp_min(0)
            rstd = torch.rsqrt(var + bn.eps)
            a = gam.detach().double() * rstd
            b = bet.detach().double() - mean * a
            tab[l - 1, :4, :C] = torch.stack([a, b, mean, rstd]).float()
            _bn_update(bn, mean, var, R)
            per.append((a, mean, rstd))
            if l >= 3:
                pos = a >= 0                            # ReLU(a z + b) is monotone in z: the pooled row is the max row iff a >= 0
                zsel = torch.where(pos, zext[0], zext[1])
                sels.append(torch.where(pos, iext[0], iext[1]))
                zsels.append(zsel)
                pooled = torch.clamp_min(tab[l - 1, 0] * zsel + tab[l - 1, 1], 0)
                if l == 3:
                    g = pooled
                    shift4 = ops.linear(g, W4g)         # (crops, 256) = g W4g^T, the concatenated half of pts_encoder_2
        rows['enc1'], rows['enc2'] = sels
        ctx.save_for_backward(x, g, pooled)
        ctx.st = (P, mode, wf, wb, W4g, shift4, tab, per, torch.stack(sels), zsels, csum)
        return pooled

    @staticmethod
    def backward(ctx, dout):
        x, g, out = ctx.saved_tensors
        P, mode, wf, wb, W4g, shift4, tab, per, sel, zsels, csum = ctx.st
        R, c0 = x.shape
        tab = tab.clone()

        def sparse(delta, l):
            """BN backward constants of a layer whose output gradient is delta at the pooled rows only"""
            a, mean, rstd = per[l - 1]
            xh = (zsels[l - 3].double() - mean) * rstd
            dbeta, dgamma = delta.sum(0), (delta * xh).sum(0)
            tab[l - 1, 4], tab[l - 1, 5] = (dbeta / R).float(), (dgamma / R).float()
            return dgamma, dbeta

        d4 = dout.double() * (out > 0)
        dgam4, dbet4 = sparse(d4, 4)
        a4, mean4, rstd4 = per[3]
        # the crop sums of dz4 in closed form: a4 (delta - P m1 - m2 sum_crop xhat4)
        S4 = a4 * (d4 - P * dbet4 / R - (dgam4 / R) * (csum - P * mean4) * rstd4)
        dW4g = S4.t() @ g.double()
        d3 = (S4 @ W4g.double()) * (g > 0)
        dgam3, dbet3 = sparse(d3, 3)
        dsel = torch.stack([d3, d4]).float()
        stats = torch.empty(512, dtype=torch.float64, device=x.device)
        slab = torch.empty(2 * C4 * C2, dtype=torch.float64, device=x.device)
        ops.crm_point_pass(5, mode, x, P, wf, wb, tab, shift4, sel, dsel, stats=stats, slab=slab)
        dW4p, dW3 = slab[:C4 * C2].view(C4, C2).clone(), slab[C4 * C2:].view(C3, C2).clone()
        dbet2, dgam2 = stats[:C2].clone(), stats[256:256 + C2].clone()
        tab[1, 4, :C2], tab[1, 5, :C2] = (dbet2 / R).float(), (dgam2 / R).float()
        ops.crm_point_pass(6, mode, x, P, wf, wb, tab, shift4, sel, dsel, stats=stats, slab=slab)
        dW2 = slab[:C2 * C1].view(C2, C1).clone()
        dbet1, dgam1 = stats[:C1].clone(), stats[256:256 + C1].clone()
        tab[0, 4, :C1], tab[0, 5, :C1] = (dbet1 / R).float(), (dgam1 / R).float()
        ops.crm_point_pass(7, mode, x, P, wf, wb, tab, shift4, sel, dsel, slab=slab)
        dW1 = slab[:C1 * c0].view(C1, c0)
        f = lambda t: t.float()                                          # noqa: E731
        dW4 = torch.cat([dW4g, dW4p], dim=1)
        return (None, None, None, None, None,
                f(dW1).view(C1, c0, 1, 1), f(dgam1), f(dbet1), f(dW2).view(C2, C1, 1, 1), f(dgam2), f(dbet2),
                f(dW3).view(C3, C2, 1, 1), f(dgam3), f(dbet3), f(dW4).view(C4, C3 + C2, 1, 1), f(dgam4), f(dbet4))


def point_encoders(module, pts):
    """ConfidencePointnet's train-mode pts_encoder_1 / pts_encoder_2 with their max-pools: pts (B, L, P, C) -> (B*L, 256)"""
    B, L, P, C = pts.shape
    if P % 64 != 0:
        raise ValueError('train-mode ConfidencePointnet needs the points per crop to be a multiple of 64 (a tile never straddles two '
                         'crops); got %d' % P)
    if C % 8 != 0 or not 8 <= C <= 64:
        raise ValueError('train-mode ConfidencePointnet needs the point dims to be a multiple of 8 in [8, 64] (the first layer\'s '
                         'reduction is staged 8 channels at a time, at most 64); got %d' % C)
    e1, e2 = module.pts_encoder_1, module.pts_encoder_2
    return CrmPointEncoders.apply(pts.reshape(B * L * P, C).contiguous(), P, module.mode, module.pooled_rows, (e1[1], e1[4], e1[7], e2[1]),
                                  e1[0].weight, e1[1].weight, e1[1].bias, e1[3].weight, e1[4].weight, e1[4].bias,
                                  e1[6].weight, e1[7].weight, e1[7].bias, e2[0].weight, e2[1].weight, e2[1].bias)


# ---- GRM: memory path and query encoder on the train-mode point layers (csrc/pointmlp_train.cu) ----------------------------------
# Unlike the CRM passes above these store each layer's pre-BatchNorm output z once (fp32, (rows, C)); BatchNorm + ReLU of a layer
# are applied when the next GEMM loads its operand.  Per layer the table is (6, C) [a, b, mean, rstd, m1, m2] (see
# include/detzero_b200.h).

def _bn_table(ps, gamma, beta, bn, R):
    """per-channel table of a layer from the sum of its per-tile partials, and the running-statistics update"""
    s = ops.pm_reduce_tiles(ps)[0]
    mean = s[0] / R
    var = (s[1] / R - mean * mean).clamp_min(0)
    rstd = torch.rsqrt(var + bn.eps)
    a = gamma.detach().double() * rstd
    b = beta.detach().double() - mean * a
    tab = torch.zeros(6, s.shape[1], dtype=torch.float32, device=s.device)
    tab[:4] = torch.stack([a, b, mean, rstd]).float()
    _bn_update(bn, mean, var, R)
    return tab, (mean, rstd)


def _set_bwd(tab, dbeta, dgamma, R):
    tab[4], tab[5] = (dbeta / R).float(), (dgamma / R).float()


def _pool(zext, iext, tab, st):
    """the pooled output of a max over each group: ReLU(a z + b) is monotone in z, so the pooled row is the max row when a >= 0 and
    the min row otherwise.  Returns (pooled (G, C), pooled row, its z)"""
    pos = tab[0] >= 0
    zsel = torch.where(pos, zext[0], zext[1])
    sel = torch.where(pos, iext[0], iext[1]).contiguous()
    return torch.clamp_min(tab[0] * zsel + tab[1], 0), sel, zsel


def _pool_bwd(dpool, pooled, zsel, st, R):
    """dH at the pooled rows and the layer's BN sums (sum dH, sum dH xhat over all rows: only the pooled rows are non-zero)"""
    mean, rstd = st
    dh = dpool.double() * (pooled > 0)
    dbeta, dgamma = dh.sum(0), (dh * (zsel.double() - mean) * rstd).sum(0)
    return dh.float().contiguous(), dbeta, dgamma


# The first layer of each path reads the raw point features (11 or 4 per point) in exact fp32 in every mode: rounded to TF32 they
# would move every z of the chain, and with it which of a track's 4096 rows is its max, for under 1 % of the FLOPs.
FIRST_MODE = _lib.DZ_F32


def _w(w):
    return w.detach().reshape(w.shape[0], -1).float().contiguous()


class GrmMemoryPath(torch.autograd.Function):
    """memory_encoder (c0 -> C1 -> C2 -> C3, max over the track's N points: g) -> memory_mlp on the concatenation of y2 and g
    (-> C4 -> 256): x (B*N, c0) -> y5 (B*N, 256).  GRM: 11 -> 128 -> 128 -> 512, cat([y2, g]) 640 -> 512 -> 256
    (geometry_transformer.py:128); PRM: 32 -> 128 -> 128 -> 256, cat([g, y2]) 384 -> 512 -> 256 (position_transformer.py:120), so
    ``glob_first`` names the concatenation order.  ``rows`` (a dict) receives the pooled row of each (track, channel) under
    'memory' and the pooled output g under 'memory_pool'.  Arguments after ``glob_first`` (``bns``: the five BatchNorm modules):
    per layer conv weight, BN weight, BN bias.  Weight gradients come back in each weight's own shape."""

    @staticmethod
    def forward(ctx, x, N, mode, rows, bns, glob_first, w1, g1, b1, w2, g2, b2, w3, g3, b3, w4, g4, b4, w5, g5, b5):
        R = x.shape[0]
        B = R // N
        W1, W2, W3, W4, W5 = (_w(w) for w in (w1, w2, w3, w4, w5))
        C2, C3 = W2.shape[0], W3.shape[0]
        if glob_first:
            W4g, W4p = W4[:, :C3].contiguous(), W4[:, C3:].contiguous()
        else:
            W4p, W4g = W4[:, :C2].contiguous(), W4[:, C2:].contiguous()
        z1, ps, _, _ = ops.pm_fwd(x, W1, FIRST_MODE)
        t1, s1 = _bn_table(ps, g1, b1, bns[0], R)
        z2, ps, _, _ = ops.pm_fwd(z1, W2, mode, t1)
        t2, s2 = _bn_table(ps, g2, b2, bns[1], R)
        z3, ps, ev, ei = ops.pm_fwd(z2, W3, mode, t2, gsize=N, ext=True)
        t3, s3 = _bn_table(ps, g3, b3, bns[2], R)
        g, sel3, zsel3 = _pool(*ops.pm_group_ext(ev, ei, B), t3, s3)
        rows['memory'], rows['memory_pool'] = sel3, g                    # the pooled output too, for the tests
        shift4 = ops.linear(g.contiguous(), W4g)                          # (B, 512) = g W4g^T, once per track
        z4, ps4, _, _ = ops.pm_fwd(z2, W4p, mode, t2, shift=shift4, gsize=N)
        t4, s4 = _bn_table(ps4, g4, b4, bns[3], R)
        zsum4 = ops.pm_reduce_tiles(ps4, B)[:, 0]                         # per-track sum of z4
        z5, ps, _, _ = ops.pm_fwd(z4, W5, mode, t4)
        t5, s5 = _bn_table(ps, g5, b5, bns[4], R)
        y5 = ops.pm_act(z5, t5)
        ctx.save_for_backward(x, z1, z2, z3, z4, z5, g)
        ctx.st = (N, mode, (W1, W2, W3, W4p, W4g, W5), (t1, t2, t3, t4, t5), (s1, s2, s3, s4, s5), sel3, zsel3, zsum4)
        ctx.glob_first, ctx.shapes = glob_first, [w.shape for w in (w1, w2, w3, w4, w5)]
        return y5

    @staticmethod
    def backward(ctx, dy5):
        x, z1, z2, z3, z4, z5, g = ctx.saved_tensors
        N, mode, (W1, W2, W3, W4p, W4g, W5), tabs, sts, sel3, zsel3, zsum4 = ctx.st
        t1, t2, t3, t4, t5 = (t.clone() for t in tabs)
        R = x.shape[0]
        B = R // N
        dh5, ps = ops.pm_dh(dy5.contiguous().float(), z5, t5)
        dbet5, dgam5 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t5, dbet5, dgam5, R)
        dh4, ps = ops.pm_dgrad([(dh5, None, None, z5, t5, W5.t().contiguous())], z4, t4, mode)
        dW5 = ops.pm_wgrad((dh5, None, None, z5, t5), z4, mode, t4)
        pg = ops.pm_reduce_tiles(ps, B)                                    # per-track sum dH4, sum dH4 xhat4
        dbet4, dgam4 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t4, dbet4, dgam4, R)
        # per-track row sums of dZ4 = a4 (dH4 - m1 - xhat4 m2): they give dg and dW4g
        mean4, rstd4 = sts[3]
        a4 = t4[0].double()
        S4 = a4 * (pg[:, 0] - N * dbet4 / R - (dgam4 / R) * (zsum4 - N * mean4) * rstd4)
        dW4g = S4.t() @ g.double()
        dh3, dbet3, dgam3 = _pool_bwd(S4 @ W4g.double(), g, zsel3, sts[2], R)
        _set_bwd(t3, dbet3, dgam3, R)
        dh2, ps = ops.pm_dgrad([(None, sel3, dh3, z3, t3, W3.t().contiguous()), (dh4, None, None, z4, t4, W4p.t().contiguous())],
                               z2, t2, mode, gsize=N)
        dW3 = ops.pm_wgrad((None, sel3, dh3, z3, t3), z2, mode, t2, gsize=N)
        dW4p = ops.pm_wgrad((dh4, None, None, z4, t4), z2, mode, t2)
        dbet2, dgam2 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t2, dbet2, dgam2, R)
        dh1, ps = ops.pm_dgrad([(dh2, None, None, z2, t2, W2.t().contiguous())], z1, t1, mode)
        dW2 = ops.pm_wgrad((dh2, None, None, z2, t2), z1, mode, t1)
        dbet1, dgam1 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t1, dbet1, dgam1, R)
        dW1 = ops.pm_wgrad((dh1, None, None, z1, t1), x, mode)
        dW4 = torch.cat([dW4g, dW4p] if ctx.glob_first else [dW4p, dW4g], dim=1)
        w1, w2, w3, w4, w5 = (t.float().view(sh) for t, sh in zip((dW1, dW2, dW3, dW4, dW5), ctx.shapes))
        f = lambda t: t.float()                                          # noqa: E731
        return (None, None, None, None, None, None,
                w1, f(dgam1), f(dbet1), w2, f(dgam2), f(dbet2), w3, f(dgam3), f(dbet3), w4, f(dgam4), f(dbet4), w5, f(dgam5), f(dbet5))


class GrmQueryEncoder(torch.autograd.Function):
    """query_encoder (GRM: 4 -> 128 -> 128 -> 256 Conv1d; PRM: 32 -> 128 -> 128 -> 256 Conv2d(1x1), BatchNorm2d) and the max over
    each group of P points: x (groups*P, c0) -> (groups, 256); ``rows`` receives the pooled rows under 'query'.  Weight gradients
    come back in each weight's own shape."""

    @staticmethod
    def forward(ctx, x, P, mode, rows, bns, w1, g1, b1, w2, g2, b2, w3, g3, b3):
        R = x.shape[0]
        W1, W2, W3 = (_w(w) for w in (w1, w2, w3))
        z1, ps, _, _ = ops.pm_fwd(x, W1, FIRST_MODE)
        t1, s1 = _bn_table(ps, g1, b1, bns[0], R)
        z2, ps, _, _ = ops.pm_fwd(z1, W2, mode, t1)
        t2, s2 = _bn_table(ps, g2, b2, bns[1], R)
        z3, ps, ev, ei = ops.pm_fwd(z2, W3, mode, t2, gsize=P, ext=True)
        t3, s3 = _bn_table(ps, g3, b3, bns[2], R)
        pooled, sel3, zsel3 = _pool(*ops.pm_group_ext(ev, ei, R // P), t3, s3)
        rows['query'] = sel3
        ctx.save_for_backward(x, z1, z2, z3, pooled)
        ctx.st = (P, mode, (W1, W2, W3), (t1, t2, t3), (s1, s2, s3), sel3, zsel3)
        ctx.shapes = [w.shape for w in (w1, w2, w3)]
        return pooled

    @staticmethod
    def backward(ctx, dout):
        x, z1, z2, z3, pooled = ctx.saved_tensors
        P, mode, (W1, W2, W3), tabs, sts, sel3, zsel3 = ctx.st
        t1, t2, t3 = (t.clone() for t in tabs)
        R = x.shape[0]
        dh3, dbet3, dgam3 = _pool_bwd(dout, pooled, zsel3, sts[2], R)
        _set_bwd(t3, dbet3, dgam3, R)
        dh2, ps = ops.pm_dgrad([(None, sel3, dh3, z3, t3, W3.t().contiguous())], z2, t2, mode, gsize=P)
        dW3 = ops.pm_wgrad((None, sel3, dh3, z3, t3), z2, mode, t2, gsize=P)
        dbet2, dgam2 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t2, dbet2, dgam2, R)
        dh1, ps = ops.pm_dgrad([(dh2, None, None, z2, t2, W2.t().contiguous())], z1, t1, mode)
        dW2 = ops.pm_wgrad((dh2, None, None, z2, t2), z1, mode, t1)
        dbet1, dgam1 = ops.pm_reduce_tiles(ps)[0]
        _set_bwd(t1, dbet1, dgam1, R)
        dW1 = ops.pm_wgrad((dh1, None, None, z1, t1), x, mode)
        w1, w2, w3 = (t.float().view(sh) for t, sh in zip((dW1, dW2, dW3), ctx.shapes))
        f = lambda t: t.float()                                          # noqa: E731
        return (None, None, None, None, None, w1, f(dgam1), f(dbet1), w2, f(dgam2), f(dbet2), w3, f(dgam3), f(dbet3))


def _check_widths(name, seq, n_layers, model='GeometryTransformer'):
    """the train-mode kernels take a stack of n_layers [Conv1d | BatchNorm1d | ReLU] or [Conv2d(1x1) | BatchNorm2d | ReLU] layers
    whose output channels are multiples of 128 (the column tile of the forward and dgrad kernels)"""
    conv = (torch.nn.Conv1d, torch.nn.Conv2d)
    convs = [m for m in seq if isinstance(m, conv)]
    widths = [m.weight.shape[0] for m in convs]
    layered = len(seq) == 3 * n_layers and all(
        isinstance(seq[3 * i], conv) and isinstance(seq[3 * i + 1], (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d))
        and isinstance(seq[3 * i + 2], torch.nn.ReLU) and all(k == 1 for k in seq[3 * i].kernel_size) for i in range(n_layers))
    if not layered or any(c % 128 for c in widths):
        raise ValueError('train-mode %s supports a %s of %d Conv + BatchNorm + ReLU layers (1x1 convs) with output channels that '
                         'are multiples of 128 (the shipped MEMORY_ENCODER / QUERY_ENCODER [128, 128], REGRESSION_MLP [512], '
                         'EMBED_DIMS 256); got output channels %s' % (model, name, n_layers, widths))


def _check_rows(what, n, model='GeometryTransformer'):
    if n % ops.PM_TILE != 0 or n <= 0:
        raise ValueError('train-mode %s needs the %s to be a positive multiple of %d (a row tile never straddles two groups); got %d'
                         % (model, what, ops.PM_TILE, n))


def grm_memory(module, mpts):
    """GeometryTransformer's train-mode memory_encoder -> max -> memory_mlp: mpts (B, N, C) -> (B*N, 256)"""
    B, N, C = mpts.shape
    _check_rows('memory points per track N', N)
    e, m = module.memory_encoder, module.memory_mlp
    _check_widths('memory_encoder', e, 3)
    _check_widths('memory_mlp', m, 2)
    return GrmMemoryPath.apply(mpts.reshape(B * N, C).contiguous(), N, module.mode, module.pooled_rows, (e[1], e[4], e[7], m[1], m[4]),
                               False, e[0].weight, e[1].weight, e[1].bias, e[3].weight, e[4].weight, e[4].bias,
                               e[6].weight, e[7].weight, e[7].bias, m[0].weight, m[1].weight, m[1].bias,
                               m[3].weight, m[4].weight, m[4].bias)


def grm_query(module, qpts):
    """GeometryTransformer's train-mode query_encoder and its max over each query's points: qpts (B, Q, P, C) -> (B*Q, 256)"""
    B, Q, P, C = qpts.shape
    _check_rows('points per query P', P)
    e = module.query_encoder
    _check_widths('query_encoder', e, 3)
    return GrmQueryEncoder.apply(qpts.reshape(B * Q * P, C).contiguous(), P, module.mode, module.pooled_rows, (e[1], e[4], e[7]),
                                 e[0].weight, e[1].weight, e[1].bias, e[3].weight, e[4].weight, e[4].bias,
                                 e[6].weight, e[7].weight, e[7].bias)


# ---- PRM: the same two paths at the PRM's widths ----------------------------------------------------------------------------------
# The kernels take the row count R as an int (every element offset inside them is 64-bit), so a PRM batch must keep B * L * P, the
# query rows, below 2^31.
MAX_ROWS = (1 << 31) - 1


def prm_memory(module, mpts):
    """PositionTransformer's train-mode memory_encoder (32 -> 128 -> 128 -> 256) -> max over the track's L * Pm rows (padded boxes
    included, as position_transformer.py:116-118 pools them) -> memory_mlp on cat([g, y2]) (384 -> 512 -> 256): mpts (B, L, Pm, C)
    -> (B*L*Pm, 256)"""
    B, L, Pm, C = mpts.shape
    N = L * Pm
    _check_rows('memory rows per track L * MEMORY_POINTS_NUM', N, 'PositionTransformer')
    if B * N > MAX_ROWS:
        raise ValueError('train-mode PositionTransformer: %d memory rows exceed the kernels\' int row count' % (B * N))
    e, m = module.memory_encoder, module.memory_mlp
    _check_widths('memory_encoder', e, 3, 'PositionTransformer')
    _check_widths('memory_mlp', m, 2, 'PositionTransformer')
    return GrmMemoryPath.apply(mpts.reshape(B * N, C).contiguous(), N, module.mode, module.pooled_rows, (e[1], e[4], e[7], m[1], m[4]),
                               True, e[0].weight, e[1].weight, e[1].bias, e[3].weight, e[4].weight, e[4].bias,
                               e[6].weight, e[7].weight, e[7].bias, m[0].weight, m[1].weight, m[1].bias,
                               m[3].weight, m[4].weight, m[4].bias)


def prm_query(module, qpts):
    """PositionTransformer's train-mode query_encoder (Conv2d(1x1) + BatchNorm2d + ReLU, 32 -> 128 -> 128 -> 256) and the max over
    each box's P points: qpts (B, L, P, C) -> (B*L, 256).  BatchNorm2d over (B, C, L, P) takes its statistics over the B*L*P rows."""
    B, L, P, C = qpts.shape
    _check_rows('query points per box P', P, 'PositionTransformer')
    if B * L * P > MAX_ROWS:
        raise ValueError('train-mode PositionTransformer: B * L * P = %d query rows exceed the kernels\' int row count (2^31 - 1)'
                         % (B * L * P))
    e = module.query_encoder
    _check_widths('query_encoder', e, 3, 'PositionTransformer')
    return GrmQueryEncoder.apply(qpts.reshape(B * L * P, C).contiguous(), P, module.mode, module.pooled_rows, (e[1], e[4], e[7]),
                                 e[0].weight, e[1].weight, e[1].bias, e[3].weight, e[4].weight, e[4].bias,
                                 e[6].weight, e[7].weight, e[7].bias)
