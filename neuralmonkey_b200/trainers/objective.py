"""Training objectives (reference: neuralmonkey/trainers/objective.py:14-110)."""
from typing import Any, List, Optional, Tuple, Union

import torch

ObjectiveWeight = Union[torch.Tensor, float, None]
Gradients = List[Tuple[torch.Tensor, torch.Tensor]]


class Objective:
    def __init__(self, name: str, decoder: Any) -> None:
        self._name = name
        self._decoder = decoder

    @property
    def decoder(self) -> Any:
        return self._decoder

    @property
    def name(self) -> str:
        return self._name

    @property
    def loss(self) -> torch.Tensor:
        raise NotImplementedError()

    @property
    def gradients(self) -> Optional[Gradients]:
        return None

    @property
    def weight(self) -> ObjectiveWeight:
        return None

    # Token-mean losses additionally expose their un-normalised sum and count so that
    # data-parallel ranks can combine them exactly (SURVEY.md 8(e)).
    @property
    def loss_sum_and_count(self) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
        return None


class CostObjective(Objective):
    """Objective over the `cost` attribute of a model part (objective.py:70-110)."""

    def __init__(self, decoder: Any, weight: ObjectiveWeight = None) -> None:
        if "cost" not in dir(decoder):
            raise TypeError("The decoder does not have the 'cost' attribute")
        Objective.__init__(self, "{} - cost".format(str(decoder)), decoder)
        self._weight = weight

    @property
    def loss(self) -> torch.Tensor:
        return getattr(self.decoder, "cost")

    @property
    def weight(self) -> ObjectiveWeight:
        return self._weight

    @property
    def loss_sum_and_count(self):
        dec = self.decoder
        if hasattr(type(dec), "loss_sum_and_count"):      # a decoder whose cost is not a token mean says how it splits
            return dec.loss_sum_and_count
        if hasattr(type(dec), "train_xent_sum") and hasattr(type(dec), "_train_mask_bm"):
            return dec.train_xent_sum, dec._train_mask_bm.sum()
        return None
