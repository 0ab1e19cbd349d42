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

from .. import ops

C1, C2, C3, C4 = 128, 128, 256, 256


def _bn_update(bn, mean, var, n):
    with torch.no_grad():
        m = bn.momentum
        bn.running_mean.mul_(1 - m).add_(mean.float(), alpha=m)
        bn.running_var.mul_(1 - m).add_((var * (n / max(n - 1, 1))).float(), alpha=m)
        bn.num_batches_tracked.add_(1)


class CrmPointEncoders(torch.autograd.Function):
    """x (crops*P, c0) -> (crops, 256).  Arguments after ``bns`` (the four BatchNorm2d modules, whose running statistics the forward
    updates): per layer the conv weight, BN weight and BN bias."""

    @staticmethod
    def forward(ctx, x, P, mode, bns, w1, g1, b1, w2, g2, b2, w3, g3, b3, w4, g4, b4):
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
        return (None, None, None, None,
                f(dW1).view(C1, c0, 1, 1), f(dgam1), f(dbet1), f(dW2).view(C2, C1, 1, 1), f(dgam2), f(dbet2),
                f(dW3).view(C3, C2, 1, 1), f(dgam3), f(dbet3), f(dW4).view(C4, C3 + C2, 1, 1), f(dgam4), f(dbet4))


def point_encoders(module, pts):
    """ConfidencePointnet's train-mode pts_encoder_1 / pts_encoder_2 with their max-pools: pts (B, L, P, C) -> (B*L, 256)"""
    B, L, P, C = pts.shape
    if P % 64 != 0:
        raise ValueError('train-mode ConfidencePointnet needs the points per crop to be a multiple of 64 (a tile never straddles two '
                         'crops); got %d' % P)
    e1, e2 = module.pts_encoder_1, module.pts_encoder_2
    return CrmPointEncoders.apply(pts.reshape(B * L * P, C).contiguous(), P, module.mode, (e1[1], e1[4], e1[7], e2[1]),
                                  e1[0].weight, e1[1].weight, e1[1].bias, e1[3].weight, e1[4].weight, e1[4].bias,
                                  e1[6].weight, e1[7].weight, e1[7].bias, e2[0].weight, e2[1].weight, e2[1].bias)
