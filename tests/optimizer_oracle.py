"""fp64 restatement of the optimizers of the reference's add_optimizer_op (DCSCN.py:379-413) other than Adam, at TF's
defaults for every argument the reference does not pass (include/dcscn_b200.h, DCSCN_OPTIMIZER_*).  Adam stays
`Oracle.adam_step` (oracle/dcscn_oracle.py); `optimizer_step` is its counterpart for the other five.

The rules follow TF1's documented training ops.  Nothing here is pinned against TensorFlow itself, which is not
available to the tests: tests/test_optimizers_cpu.py pins gd, momentum, adagrad and adadelta against torch.optim in
float64, and rmsprop (whose torch.optim version differs) against a literal loop of the formula."""
import numpy as np

KINDS = ("gd", "momentum", "adadelta", "adagrad", "rmsprop")
# initial value of each slot, in the engine's slot order
SLOT_INIT = {"gd": (), "momentum": (0.0,), "adadelta": (0.0, 0.0), "adagrad": (0.1,), "rmsprop": (1.0, 0.0)}
ADADELTA_RHO, ADADELTA_EPS = 0.95, 1e-8
RMSPROP_RHO, RMSPROP_EPS = 0.9, 1e-10


def init_slots(kind, weights):
    return {n: [np.full(np.shape(w), v, np.float64) for v in SLOT_INIT[kind]] for n, w in weights.items()}


def update(kind, w, g, slots, lr, momentum=0.9):
    """One update of weight array `w` with clipped gradient `g`; returns (new w, new slots), all float64."""
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
    raise ValueError(kind)


def optimizer_step(orc, kind, grads, slots, lr, momentum=0.9):
    """`Oracle.adam_step` for the other optimizers: updates orc.w (in its dtype) and `slots` (float64) in place."""
    for n, g in grads.items():
        w, slots[n] = update(kind, orc.w[n], g, slots[n], lr, momentum)
        orc.w[n] = w.astype(orc.w[n].dtype)
