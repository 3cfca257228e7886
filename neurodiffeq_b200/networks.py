"""Network definitions accepted by the fused path (reference neurodiffeq/networks.py:6-70, 142-152).

``FCNN`` keeps the reference's module layout -- an ``nn.Sequential`` called ``NN`` of ``Linear, actv, ..., Linear`` with
parameters at ``NN.{0,2,4,...}.{weight,bias}`` -- so state dicts, optimizers, checkpoints and ``deepcopy`` of user code
keep working; the CUDA engine reads the weights of exactly this structure (any ``nn.Sequential`` alternating
``nn.Linear`` with ``nn.Tanh`` / ``SinActv`` / ``nn.Sigmoid`` / ``nn.SiLU`` / ``nn.ELU`` (alpha = 1) is accepted, see
``tracing.NetDescription``).
"""
from warnings import warn

import torch
import torch.nn as nn


class SinActv(nn.Module):
    """sin activation (reference networks.py:142-152)."""

    def forward(self, input_):
        return torch.sin(input_)


class FCNN(nn.Module):
    """Fully connected network; defaults (32, 32) hidden units and tanh like the reference (networks.py:52-53)."""

    def __init__(self, n_input_units=1, n_output_units=1, n_hidden_units=None, n_hidden_layers=None,
                 actv=nn.Tanh, hidden_units=None):
        super().__init__()
        if n_hidden_units is not None or n_hidden_layers is not None:  # deprecated pair, reference networks.py:32-50
            n_hidden_units = 32 if n_hidden_units is None else n_hidden_units
            n_hidden_layers = 1 if n_hidden_layers is None else n_hidden_layers
            if hidden_units is None:
                hidden_units = tuple(n_hidden_units for _ in range(n_hidden_layers + 1))
                warn(f"`n_hidden_units` and `n_hidden_layers` are deprecated, pass `hidden_units={hidden_units}`",
                     FutureWarning)
            else:
                warn(f"Ignoring `n_hidden_units` and `n_hidden_layers` in favor of `hidden_units={hidden_units}`",
                     FutureWarning)
        if hidden_units is None:
            hidden_units = (32, 32)
        hidden_units = tuple(hidden_units)
        widths = (n_input_units,) + hidden_units
        layers = []
        for fan_in, fan_out in zip(widths[:-1], widths[1:]):
            layers.append(nn.Linear(fan_in, fan_out))
            layers.append(actv())
        layers.append(nn.Linear(widths[-1], n_output_units))
        self.NN = nn.Sequential(*layers)

    def forward(self, t):
        return self.NN(t)


# ----------------------------------------------------------------------------------------------------------------------
# The remaining modules of the reference's networks.py: ordinary torch modules with the reference's semantics.  The fused
# engine runs Resnet (FCNN body on the kernels, shortcut inside the residual program); MonomialNN / Swish / APTx have no jet
# rule in the kernels yet and a solver built with them says so.
# ----------------------------------------------------------------------------------------------------------------------
def _scalar(value, trainable):
    """a python float, or a 0-dim Parameter when the activation's scalars are to be learned"""
    value = float(value)
    return nn.Parameter(torch.tensor(value)) if trainable else value


class Resnet(nn.Module):
    """FCNN plus a bias-free linear shortcut from the inputs to the outputs (reference networks.py:73-106); the
    sub-modules keep the reference's names ``residual`` and ``skip_connection`` so that state dicts are interchangeable."""

    def __init__(self, n_input_units=1, n_output_units=1, n_hidden_units=None, n_hidden_layers=None, actv=nn.Tanh,
                 hidden_units=(32, 32)):
        super().__init__()
        body = dict(n_hidden_units=n_hidden_units, n_hidden_layers=n_hidden_layers, actv=actv, hidden_units=hidden_units)
        self.residual = FCNN(n_input_units, n_output_units, **body)
        self.skip_connection = nn.Linear(n_input_units, n_output_units, bias=False)

    def forward(self, t):
        shortcut = self.skip_connection(t)
        return shortcut + self.residual(t)


class MonomialNN(nn.Module):
    """Parameter-free feature map: the columns of ``x`` raised to each of ``degrees`` (an int n means 1..n), side by
    side -> ``(n_samples, n_inputs * len(degrees))`` (reference networks.py:109-139)."""

    def __init__(self, degrees):
        super().__init__()
        powers = tuple(range(1, degrees + 1)) if isinstance(degrees, int) else tuple(degrees)
        if not powers:
            raise ValueError("No degrees used, check `degrees` argument again")
        if any(p == 0 for p in powers):
            warn("One of the degrees is 0 which might introduce redundant features")
        if len(powers) != len(set(powers)):
            warn(f"Duplicate degrees found: {powers}")
        self.degrees = powers

    def forward(self, x):
        return torch.cat(tuple(torch.pow(x, p) for p in self.degrees), dim=1)

    def extra_repr(self):
        return f"degrees={self.degrees}"

    def __repr__(self):
        return f"{type(self).__name__}({self.extra_repr()})"


class Swish(nn.Module):
    """swish(x) = x / (1 + exp(-beta x)); ``beta`` may be trainable (reference networks.py:155-174)."""

    def __init__(self, beta=1.0, trainable=False):
        super().__init__()
        self.trainable = trainable
        self.beta = _scalar(beta, trainable)

    def forward(self, x):
        gate = torch.sigmoid(x * self.beta)
        return gate * x


class APTx(nn.Module):
    """APTx(x) = (alpha + tanh(beta x)) gamma x, a cheaper look-alike of MISH; the three scalars may be trainable
    (reference networks.py:177-208)."""

    def __init__(self, alpha=1.0, beta=1.0, gamma=0.5, trainable=False):
        super().__init__()
        self.trainable = trainable
        self.alpha, self.beta, self.gamma = (_scalar(v, trainable) for v in (alpha, beta, gamma))

    def forward(self, x):
        return self.gamma * x * (torch.tanh(x * self.beta) + self.alpha)
