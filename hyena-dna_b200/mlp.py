"""The block MLP of the HyenaDNA backbone: fc1 -> GELU -> fc2 (SURVEY.md S8 f1, the MLP after the mixer).

Mirrors flash-attention/flash_attn/modules/mlp.py:13-30 (``Mlp``), which src/models/sequence/long_conv_lm.py:102-123
(create_mlp_cls) builds with ``hidden_features = d_inner = 4 * d_model`` and ``activation=partial(F.gelu,
approximate="tanh")``: same constructor keywords, attribute names and state_dict keys (``fc1.weight``, ``fc1.bias``,
``fc2.weight``, ``fc2.bias``), so a reference checkpoint's ``backbone.layers.N.mlp.*`` entries load unchanged.

With the projections on this library's wgmma kernels (ops.proj_mode() == "tc", the default) the whole MLP is one autograd
node (ops.MlpFn) whose GELU and GELU gradient are fused into the GEMMs; it saves one hidden-sized tensor.  Under the
library GEMM modes (HYENA_B200_PROJ=lt / torch, or torch.backends.cuda.matmul.allow_tf32) it is the reference's own
F.linear + F.gelu composition, exactly as the projections of HyenaOperator follow that switch.  There is no CPU path.

When no gradient is needed, a row count L > 4 that is not a multiple of 4 (a packed batch, whose L is its token count) is
zero-padded to one: the hidden activation's channel stride is then a multiple of 4 and fc2 reads it on the vector path.
Each output element sums over the features in the same order whatever L is, so the real rows keep their bits.  Training
keeps L as it is: the weight-gradient sums over L would change order.
"""
import torch
import functools

import torch.nn as nn
import torch.nn.functional as F

from . import ops
from ._lib import HyenaB200Error


def _gelu_approximate(activation):
    """'tanh' / 'none' for F.gelu and partial(F.gelu, approximate=...); None for anything else."""
    if activation is F.gelu:
        return "none"
    if isinstance(activation, functools.partial) and activation.func is F.gelu and not activation.args \
            and set(activation.keywords) <= {"approximate"}:
        approximate = activation.keywords.get("approximate", "none")
        return approximate if approximate in ("tanh", "none") else None
    return None


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, activation=F.gelu, bias1=True, bias2=True,
                 return_residual=False, device=None, dtype=None):
        factory_kwargs = {"device": device, "dtype": dtype}
        super().__init__()
        self.approximate = _gelu_approximate(activation)
        if self.approximate is None:
            raise HyenaB200Error(f"Mlp: activation {activation!r} is not fused on sm_90a; supported: F.gelu and "
                                 "partial(F.gelu, approximate='tanh' | 'none')")
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features * 4
        self.return_residual = return_residual
        self.fc1 = nn.Linear(in_features, hidden_features, bias=bias1, **factory_kwargs)
        self.activation = activation
        self.fc2 = nn.Linear(hidden_features, out_features, bias=bias2, **factory_kwargs)

    def forward(self, x):
        if not x.is_cuda:
            raise HyenaB200Error("Mlp (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        if ops.proj_mode() == "tc":
            shape = x.shape
            x3 = x.reshape(-1, shape[-2], shape[-1]) if x.dim() >= 2 else x.reshape(1, 1, -1)
            L = x3.shape[1]
            pad = (-L) % 4 if L > 4 and not self._needs_grad(x) else 0
            if pad:
                x3 = F.pad(x3, (0, 0, 0, pad))
            y = ops.MlpFn.apply(x3, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, self.approximate)
            if pad:
                y = y[:, :L]
            y = y.reshape(*shape[:-1], y.shape[-1])
        else:
            y = self.fc2(self.activation(self.fc1(x)))
        return y if not self.return_residual else (y, x)

    def _needs_grad(self, x):
        return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))
