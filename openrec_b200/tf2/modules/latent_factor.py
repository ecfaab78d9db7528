"""LatentFactor -- mirrors openrec/tf2/modules/latent_factor.py:4-23 on liborx."""
import torch

from ... import native as N
from ...tfshim.core import Tensor, convert
from ...tfshim.keras.layers import Embedding


class LatentFactor(Embedding):
    """Embedding table [num_instances, dim]; U(-0.05, 0.05) init unless zero_init (latent_factor.py:6-15).
    Calling it gathers rows (orx_gather); ``variables[0]`` is the table (bpr.py:42).

    ``dtype="bfloat16"`` stores the table in bfloat16: the float32 initial values rounded to nearest even, optimizer
    slots in float32, updates rounded stochastically by the fused BPR / UCML step.  A lookup returns float32 rows."""

    def __init__(self, num_instances, dim, zero_init=False, name=None, dtype="float32"):
        if dtype not in ("float32", "bfloat16"):
            raise ValueError(f"LatentFactor dtype must be 'float32' or 'bfloat16', got {dtype!r}")
        super().__init__(input_dim=num_instances, output_dim=dim,
                         embeddings_initializer="zeros" if zero_init else "uniform", name=name)
        if dtype == "bfloat16":
            self.embeddings.t = self.embeddings.t.to(torch.bfloat16)

    def call(self, ids):
        if self.embeddings.t.dtype != torch.bfloat16:
            return super().call(ids)
        # a bf16 row of even width is a float32 row of half the width, bit for bit: gather those, then widen
        if self.output_dim % 2:
            raise NotImplementedError("looking up a bfloat16 LatentFactor needs an even dim")
        ids_t = convert(ids).t
        tab = self.embeddings.t.view(torch.float32)
        rows = N.engine().gather(tab, ids_t if ids_t.dtype == torch.int64 else ids_t.to(torch.int32))
        rows = rows.view(torch.bfloat16).float()
        return Tensor(rows.reshape(tuple(ids_t.shape) + (self.output_dim,)))

    def censor(self, censor_id):
        """rows of the unique ids <- row / max(||row||, 0.1)  (latent_factor.py:17-23), in place (a bf16 table:
        computed in float32, stored rounded to nearest even)."""
        if self.embeddings.t.dtype == torch.bfloat16:
            N.engine().censor_bf16(self.embeddings.t, convert(censor_id).t, 0.1)
        else:
            N.engine().censor(self.embeddings.t, convert(censor_id).t, 0.1)
        return self.embeddings
