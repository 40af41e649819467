"""fp64 restatement of the optimizers of the reference's add_optimizer_op (DCSCN.py:379-413), at TF's defaults for every
argument the reference does not pass (include/dcscn_b200.h, DCSCN_OPTIMIZER_*).  `update` holds one element-wise step of
each rule, Adam included; `optimizer_step` is the counterpart of `Oracle.adam_step` (oracle/dcscn_oracle.py) for the
other five.

The rules follow TF1's documented training ops.  Nothing here is pinned against TensorFlow itself, which is not
available to the tests: tests/test_optimizers_cpu.py pins gd, momentum, adagrad and adadelta against torch.optim in
float64, rmsprop (whose torch.optim version differs) against a literal loop of the formula, and adam against
`Oracle.adam_step` and a literal loop (torch.optim.Adam adds epsilon after the bias correction: not TF's rule)."""
import numpy as np

KINDS = ("gd", "momentum", "adadelta", "adagrad", "rmsprop")
# initial value of each slot, in the engine's slot order
SLOT_INIT = {"gd": (), "momentum": (0.0,), "adadelta": (0.0, 0.0), "adagrad": (0.1,), "rmsprop": (1.0, 0.0),
             "adam": (0.0, 0.0)}
ADADELTA_RHO, ADADELTA_EPS = 0.95, 1e-8
RMSPROP_RHO, RMSPROP_EPS = 0.9, 1e-10


def init_slots(kind, weights):
    return {n: [np.full(np.shape(w), v, np.float64) for v in SLOT_INIT[kind]] for n, w in weights.items()}


def adam_lr(lr, t, beta1, beta2):
    """tf.train.AdamOptimizer's step size at update t (1 for the first): lr * sqrt(1 - beta2^t) / (1 - beta1^t)."""
    return lr * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)


def update(kind, w, g, slots, lr, momentum=0.9, t=1, beta1=0.9, beta2=0.999, epsilon=1e-8):
    """One update of weight array `w` with clipped gradient `g`; returns (new w, new slots), all float64.  Adam's update
    t (1 for the first) and its beta1 / beta2 / epsilon are used by "adam" only, momentum by momentum and rmsprop."""
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    s = [np.asarray(a, np.float64) for a in slots]
    if kind == "gd":
        return w - lr * g, []
    if kind == "momentum":
        a = momentum * s[0] + g
        return w - lr * a, [a]
    if kind == "adagrad":
        acc = s[0] + g * g
        return w - lr * g / np.sqrt(acc), [acc]
    if kind == "adadelta":
        rho, eps = ADADELTA_RHO, ADADELTA_EPS
        acc = rho * s[0] + (1 - rho) * g * g
        u = np.sqrt(s[1] + eps) / np.sqrt(acc + eps) * g          # the OLD accum_update
        return w - lr * u, [acc, rho * s[1] + (1 - rho) * u * u]
    if kind == "rmsprop":
        rho, eps = RMSPROP_RHO, RMSPROP_EPS
        ms = s[0] + (g * g - s[0]) * (1 - rho)
        mom = momentum * s[1] + lr * g / np.sqrt(ms + eps)         # epsilon inside the square root
        return w - mom, [ms, mom]
    if kind == "adam":
        m = beta1 * s[0] + (1 - beta1) * g
        v = beta2 * s[1] + (1 - beta2) * g * g
        return w - adam_lr(lr, t, beta1, beta2) * m / (np.sqrt(v) + epsilon), [m, v]   # epsilon outside the root
    raise ValueError(kind)


def optimizer_step(orc, kind, grads, slots, lr, momentum=0.9):
    """`Oracle.adam_step` for the other optimizers: updates orc.w (in its dtype) and `slots` (float64) in place."""
    for n, g in grads.items():
        w, slots[n] = update(kind, orc.w[n], g, slots[n], lr, momentum)
        orc.w[n] = w.astype(orc.w[n].dtype)
