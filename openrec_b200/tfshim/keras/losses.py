"""tf.keras.losses used by the reference's model files (dlrm.py:52-55, gmf.py:20).  The liborx
recommenders compute their losses inside liborx; these callables exist for user-side evaluation
glue on already-materialised tensors."""
from __future__ import annotations

import torch

from ..core import Tensor, convert


class MeanSquaredError:
    def __call__(self, y_true, y_pred):
        p = convert(y_pred).t.to(torch.float32)
        return Tensor(((convert(y_true).t.to(torch.float32) - p) ** 2).mean())


class BinaryCrossentropy:
    def __init__(self, from_logits=False):
        self.from_logits = from_logits

    def __call__(self, y_true, y_pred):
        y = convert(y_true).t.to(torch.float32)
        z = convert(y_pred).t.to(torch.float32)
        if self.from_logits:
            return Tensor((torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))).mean())
        eps = 1e-7
        p = torch.clamp(z, eps, 1 - eps)
        return Tensor(-(y * torch.log(p + eps) + (1 - y) * torch.log(1 - p + eps)).mean())
