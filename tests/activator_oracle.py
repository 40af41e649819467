"""The fp64 oracle (oracle/dcscn_oracle.py) for every --activator value (helper/tf_graph.py:77-102).

Each of CNN1..CNNL, A1, B1 and B2 computes z = conv + bias, h = f(z), then dropout; Up-PS, Up-PS2 and R-CNN1 stay
linear.  Only prelu creates a variable.  The gradients follow TensorFlow's gradient ops, also at z = 0, where two of
them differ from torch autograd: leaky_relu = tf.maximum(z, 0.1 z) passes the gradient to z where z >= 0.1 z (slope 1
at 0, torch.maximum splits a tie in half), and SeluGrad takes lambda at 0 (F.selu's backward takes lambda * alpha).
relu (ReluGrad: 0 at 0), sigmoid and tanh match torch."""
import numpy as np
import torch

import dcscn_oracle as O

ACTIVATORS = ("prelu", "relu", "leaky_relu", "sigmoid", "tanh", "selu")
SELU_SCALE = 1.0507009873554805
SELU_ALPHA = 1.6732632423543772
LEAKY = float(np.float32(0.1))        # tf.maximum(z, 0.1 * z) on fp32 tensors: the constant is the fp32 0.1


def activated(scope):
    return scope.startswith("CNN") or scope in ("A1", "B1", "B2")


def variable_names(cfg, activator):
    """The variables the reference's tf.train.Saver writes for this flag: no slope variable but for prelu."""
    names = O.variable_names(cfg)
    return names if activator == "prelu" else [n for n in names if "/prelu/" not in n]


def he_init_weights(cfg, activator, seed=0):
    w = O.he_init_weights(cfg, seed=seed)
    return {n: w[n] for n in variable_names(cfg, activator)}


class _Relu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        h = torch.clamp_min(z, 0.0)
        ctx.save_for_backward(h)
        return h

    @staticmethod
    def backward(ctx, g):
        h, = ctx.saved_tensors
        return g * (h > 0).to(g.dtype)                  # ReluGrad: 0 at z = 0


class _LeakyRelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        ctx.save_for_backward(z)
        return torch.where(z >= LEAKY * z, z, LEAKY * z)

    @staticmethod
    def backward(ctx, g):
        z, = ctx.saved_tensors
        return torch.where(z >= LEAKY * z, g, LEAKY * g)  # Maximum's gradient: 1 at z = 0


class _Selu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        h = torch.where(z < 0, SELU_SCALE * SELU_ALPHA * torch.expm1(z), SELU_SCALE * z)
        ctx.save_for_backward(h)
        return h

    @staticmethod
    def backward(ctx, g):
        h, = ctx.saved_tensors
        return torch.where(h < 0, g * (h + SELU_SCALE * SELU_ALPHA), g * SELU_SCALE)   # SeluGrad: lambda at z = 0


def activate(z, activator):
    """f(z) for every activator but prelu (whose slope is a variable: dcscn_oracle.Oracle._layer)."""
    if activator == "relu":
        return _Relu.apply(z)
    if activator == "leaky_relu":
        return _LeakyRelu.apply(z)
    if activator == "sigmoid":
        return torch.sigmoid(z)                         # SigmoidGrad = g y (1 - y), autograd's rule
    if activator == "tanh":
        return torch.tanh(z)                            # TanhGrad = g (1 - y^2), autograd's rule
    if activator == "selu":
        return _Selu.apply(z)
    raise NameError("Not implemented activator:%s" % activator)


class Oracle(O.Oracle):
    """dcscn_oracle.Oracle with `activator` in place of PReLU.  For the other activators the base class runs each
    activated layer as a linear one (its table entry without the PReLU flag, so conv + bias and no dropout) and this
    class applies f and then the dropout of tf_graph.py:124-130."""

    def __init__(self, cfg, weights, activator, dtype=torch.float64):
        super().__init__(cfg, weights, dtype)
        self.activator = activator
        if activator != "prelu":
            self.table = [e[:5] + (False,) for e in self.table]

    def _layer(self, scope, x, params=None, keep_prob=1.0, masks=None):
        if self.activator == "prelu" or not activated(scope):
            return super()._layer(scope, x, params, keep_prob, masks)
        h = activate(super()._layer(scope, x, params), self.activator)
        if keep_prob < 1.0:
            m = masks[scope]
            h = h * (m if torch.is_tensor(m) else O._t(m, self.dtype)) * (1.0 / keep_prob)
        return h

    def trainable_names(self):
        return variable_names(self.cfg, self.activator)
