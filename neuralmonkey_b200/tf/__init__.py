"""`tf.` names that Neural Monkey INI files reference literally
(config/builder.py:35-41 resolves `tf.` through the tensorflow module; e.g.
tests/transformer.ini:97-102 `tf.contrib.opt.LazyAdamOptimizer`, tests/small.ini:68-80
`tf.random_uniform_initializer`).  Only those names exist here: optimizers are plain
hyper-parameter records consumed by the K13 kernel, initialisers are arena initialisers.
"""
from types import SimpleNamespace

from neuralmonkey_b200.params import (constant_initializer, normal_initializer, ones_initializer,
                                      orthogonal_initializer as _ortho, uniform_initializer,
                                      variance_scaling_initializer as _vs, zeros_initializer)


class Optimizer:
    """Hyper-parameters of an optimizer; the update itself is nm_clip_adam_step."""
    lazy = False

    def __init__(self, learning_rate=0.001, beta1: float = 0.9, beta2: float = 0.999,
                 epsilon: float = 1e-8, use_locking: bool = False, name: str = "Adam") -> None:
        self.learning_rate = learning_rate  # float or callable(global_step) -> float
        self.beta1 = beta1
        self.beta2 = beta2
        self.epsilon = epsilon
        self.name = name
        # updates THIS optimizer has applied: tf.train.AdamOptimizer's beta1_power / beta2_power accumulators
        # are its own non-slot variables, multiplied once per apply_gradients call of this object - the bias
        # correction follows them, not the global step the trainers of an experiment share
        self.steps = 0

    def lr_at(self, global_step: int) -> float:
        lr = self.learning_rate
        return float(lr(global_step)) if callable(lr) else float(lr)


class AdamOptimizer(Optimizer):
    """tf.train.AdamOptimizer."""


class LazyAdamOptimizer(Optimizer):
    """tf.contrib.opt.LazyAdamOptimizer: rows of embedding matrices that received no
    gradient are left untouched (moments included)."""
    lazy = True


class AdadeltaOptimizer(Optimizer):
    """tf.train.AdadeltaOptimizer; the update is nm_clip_adadelta_step (the two accumulators take the two
    optimizer slots of the arena)."""

    def __init__(self, learning_rate=0.001, rho: float = 0.95, epsilon: float = 1e-8, use_locking: bool = False,
                 name: str = "Adadelta") -> None:
        Optimizer.__init__(self, learning_rate, epsilon=epsilon, use_locking=use_locking, name=name)
        self.rho = rho


def random_uniform_initializer(minval=0.0, maxval=1.0, seed=None, dtype=None):
    return uniform_initializer(minval, maxval)


def random_normal_initializer(mean=0.0, stddev=1.0, seed=None, dtype=None):
    return normal_initializer(stddev=stddev, mean=mean)


def orthogonal_initializer(gain=1.0, seed=None, dtype=None):
    return _ortho()


def variance_scaling_initializer(scale=1.0, mode="fan_in", distribution="normal", seed=None,
                                 dtype=None):
    dist = "uniform" if distribution == "uniform" else "normal"
    return _vs(scale=scale, mode=mode, distribution=dist)


train = SimpleNamespace(AdamOptimizer=AdamOptimizer, AdadeltaOptimizer=AdadeltaOptimizer, Optimizer=Optimizer)
contrib = SimpleNamespace(opt=SimpleNamespace(LazyAdamOptimizer=LazyAdamOptimizer))
tanh = "tanh"
sigmoid = "sigmoid"
nn = SimpleNamespace(relu="relu", tanh="tanh", sigmoid="sigmoid")
