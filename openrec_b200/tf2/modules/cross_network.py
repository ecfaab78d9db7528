"""CrossNetwork -- the DCN-v2 cross network (Wang et al., 2021), as TensorFlow Recommenders' ``tfrs.layers.dcn.Cross``
stacked ``num_layers`` deep.  With x0 the [B, W] input, layer l computes

    y_l = U_l (V_l^T x_l) + b_l      (projection_dim = r: V_l [W, r] without bias, U_l [r, W], b_l [W])
    y_l = K_l x_l + b_l              (projection_dim = None: K_l [W, W], b_l [W])
    x_{l+1} = x0 * y_l + x_l

Kernels follow the Keras [in, out] convention and are initialised like the shim's Dense (glorot-uniform, zero biases);
TFRS draws them from a truncated normal instead.  The projections run on the Dense-layer GEMM (orx_mlp_layer_fwd), the
element-wise step on orx_cross_fwd.  DLRM(arch_interaction_op="cross") trains it in its fused step."""
import torch

from ... import native as N
from ...tfshim.core import Tensor, Variable, convert, device
from ...tfshim.keras.layers import Layer, next_seed


class CrossNetwork(Layer):
    def __init__(self, num_layers, projection_dim=None, name=None):
        super().__init__(name=name)
        if int(num_layers) != num_layers or num_layers < 1:
            raise ValueError(f"num_layers must be an integer >= 1, got {num_layers!r}")
        if projection_dim is not None and (int(projection_dim) != projection_dim or projection_dim < 1):
            raise ValueError(f"projection_dim must be None or an integer >= 1, got {projection_dim!r}")
        self.num_layers = int(num_layers)
        self.projection_dim = None if projection_dim is None else int(projection_dim)
        self.width = None
        self.built = False
        self._proj = []        # per layer: [(kernel, bias or None)] Variables, applied in order

    def _var(self, t, name):
        v = Variable.__new__(Variable)
        v.t, v.trainable, v.name = t, True, f"{self.name}/{name}"
        return v

    def _kernel(self, n_in, n_out, name):
        lim = (6.0 / (n_in + n_out)) ** 0.5                     # glorot-uniform, as Dense
        t = torch.empty((n_in, n_out), dtype=torch.float32, device=device())
        N.engine().fill_uniform(t, -lim, lim, next_seed())
        return self._var(t, name)

    def build(self, width):
        """Create the variables for a [B, width] input (once; a later call must pass the same width)."""
        width = int(width)
        if self.built:
            if width != self.width:
                raise ValueError(f"CrossNetwork was built for width {self.width}, got {width}")
            return
        proj = []
        for l in range(self.num_layers):
            pre = f"cross_layer_{l}"
            bias = self._var(torch.zeros(width, dtype=torch.float32, device=device()), f"{pre}/bias")
            if self.projection_dim is None:
                proj.append([(self._kernel(width, width, f"{pre}/kernel"), bias)])
            else:
                v = self._kernel(width, self.projection_dim, f"{pre}/v")
                proj.append([(v, None), (self._kernel(self.projection_dim, width, f"{pre}/u"), bias)])
        self._proj, self.width, self.built = proj, width, True

    def projections(self):
        """Per layer, the [(kernel, bias or None)] Variables in the order they are applied."""
        return [list(p) for p in self._proj]

    def _own_variables(self):
        return [v for p in self._proj for pair in p for v in pair if v is not None]

    def call(self, x0):
        """x0 [B, width] -> x_L [B, width] (forward only)."""
        from .. import mlp_ops
        x0 = convert(x0).t.to(torch.float32).contiguous()
        self.build(x0.shape[1])
        eng, x = N.engine(), x0
        for p in self._proj:
            h = x
            for w, b in p:
                h = mlp_ops.dense_forward(h, w.t, None if b is None else b.t, None)
            nxt = torch.empty_like(x0)
            eng.cross_fwd(x0, x, h, nxt)
            x = nxt
        return Tensor(x)
