"""Golden vectors for CRM training: the reference's own ConfidencePointnet (refining/detzero_refine/models/modules/
confidence_pointnet.py, unmodified) run on CPU in float64 and train mode, one forward + get_loss + backward, with seeded weights
(weights.load_seeded), inputs crm_inputs(SEED, B=2) and seeded IoU labels (-1 past each track's box_num).

Stored: the three losses; the full gradients of pts_encoder_1 / pts_encoder_2; every BatchNorm's running statistics after the step;
for every other parameter its gradient's sum of squares and its dot product with a seeded probe tensor (oracle.crm_train_ref.probe)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import ref_import  # noqa: E402

ref_import.install()
from oracle import crm_train_ref  # noqa: E402
from oracle import refine_inputs as ri  # noqa: E402
from oracle import weights  # noqa: E402

SEED = 7301
B = 2


def golden_crm_train():
    from detzero_refine.models.modules.confidence_pointnet import ConfidencePointnet
    torch.manual_seed(0)
    crm = ConfidencePointnet(ri.crm_cfg(), 32, 32)
    weights.load_seeded(crm, SEED)
    crm = crm.double().train()
    inp = ri.crm_inputs(SEED, B=B)
    L = inp['conf_points'].shape[1]
    iou = crm_train_ref.crm_train_iou(SEED, B, L)
    d = {'conf_points': inp['conf_points'].double(), 'iou': iou.double()}
    crm(d)
    loss, tb = crm.get_loss({})
    loss.backward()
    out = {'loss.' + k: np.float64(tb[k].item()) for k in ('bin_cls_loss', 'iou_loss', 'confidence_loss')}
    for k, p in crm.named_parameters():
        gr = p.grad.detach()
        if k.startswith(('pts_encoder_1.', 'pts_encoder_2.')):
            out['grad.' + k] = gr.float().numpy()
        else:
            out['gsq.' + k] = np.float64((gr * gr).sum().item())
            out['gdot.' + k] = np.float64((gr * crm_train_ref.probe(k, gr.shape, SEED)).sum().item())
    for k, v in crm.state_dict().items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked')):
            out['bn.' + k] = v.numpy()
    np.savez_compressed(os.path.join(HERE, 'crm_train.npz'), **out)
    print('crm_train.npz:', len(out), 'arrays,', os.path.getsize(os.path.join(HERE, 'crm_train.npz')), 'bytes;', {k: out[k] for k in out if k.startswith('loss.')})


if __name__ == '__main__':
    golden_crm_train()
