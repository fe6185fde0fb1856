"""Highway layer (reference: neuralmonkey/nn/highway.py:6-60), with the reference's ReLU activation:

    T = sigmoid(x W_T + b_T),  H = relu(x W_H + b_H),  y = H T + x (1 - T)

The two products run on the dense GEMM (`ops.linear`), the gate on `ops.highway_gate`.  The variables of the owning
part are `<scope>/weight_H`, `bias_H`, `weight_T`, `bias_T`; both biases start at -1.  The reference gets the weights
with `get_variable` and no initializer, and neither its variable scope nor the experiment supplies one, so they take
TF's `get_variable` default, glorot uniform (`fan_avg`, uniform)."""
import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.params import constant_initializer, variance_scaling_initializer

# tf.get_variable's default initializer
_GLOROT = variance_scaling_initializer(1.0, "fan_avg", "uniform")


def declare_highway(part, scope: str, size: int) -> None:
    for gate in ("H", "T"):
        part.declare("{}/weight_{}".format(scope, gate), [size, size], _GLOROT)
        part.declare("{}/bias_{}".format(scope, gate), [size], constant_initializer(-1.0))


def highway(part, scope: str, x: torch.Tensor) -> torch.Tensor:
    """One highway layer over x [N, size] with the variables `declare_highway` declared under `scope`."""
    zh = ops.linear(x, part.var(scope + "/weight_H"), part.var(scope + "/bias_H"))
    zt = ops.linear(x, part.var(scope + "/weight_T"), part.var(scope + "/bias_T"))
    return ops.highway_gate(zh, zt, x)
