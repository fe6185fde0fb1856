"""Gradient-reversal views of encoder-like objects (reference: neuralmonkey/model/gradient_reversal.py): the same
states, but the gradient that flows back through the view is negated, for adversarial objectives (tests/
classifier.ini trains a second classifier through one).  Dependencies are handled as in
`model/gradient_blocking.py`: the view owns nothing, the wrapped object stays reachable through `dependencies`,
and the view re-reads the wrapped object's per-batch tensors at every access (it is fed nothing, so it caches
nothing)."""
from typing import Any, List

import torch

from neuralmonkey_b200.model.stateful import SpatialStateful, Stateful, TemporalStateful
from neuralmonkey_b200.typecheck import check_type


class _Reverse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, grad):
        return -grad


def reverse_gradient(x: torch.Tensor) -> torch.Tensor:
    """Identity forward, negated gradient backward."""
    return _Reverse.apply(x)


def _same(attribute: str) -> property:
    return property(lambda view: getattr(view._reversed_object, attribute))  # pylint: disable=protected-access


class _ReversalView:
    _interface = object  # type: Any

    def __init__(self, reversed_object) -> None:
        check_type("reversed_object", reversed_object, self._interface)
        self._reversed_object = reversed_object

    dimension = _same("dimension")

    @property
    def output_dimension(self) -> int:
        obj = self._reversed_object
        width = getattr(obj, "output_dimension", None)
        return obj.dimension if width is None else width

    @property
    def dependencies(self) -> List[str]:
        return super().dependencies + ["_reversed_object"]


class StatefulView(_ReversalView, Stateful):
    """Provides an adversarial view of a `Stateful` object."""
    _interface = Stateful

    @property
    def output(self) -> torch.Tensor:
        return reverse_gradient(self._reversed_object.output)


class TemporalStatefulView(_ReversalView, TemporalStateful):
    """Provides an adversarial view of a `TemporalStateful` object."""
    _interface = TemporalStateful
    temporal_mask = _same("temporal_mask")

    @property
    def temporal_states(self) -> torch.Tensor:
        return reverse_gradient(self._reversed_object.temporal_states)


class SpatialStatefulView(_ReversalView, SpatialStateful):
    """Provides an adversarial view of a `SpatialStateful` object."""
    _interface = SpatialStateful
    spatial_mask = _same("spatial_mask")

    @property
    def spatial_states(self) -> torch.Tensor:
        return reverse_gradient(self._reversed_object.spatial_states)
