"""Multilayer perceptron (reference: neuralmonkey/nn/mlp.py): `multilayer_projection` under
`<name>/deep_output_mlp`, then the dense `<name>/classification_layer`.  It is not a model part: its variables
belong to the part that owns it (`Classifier`)."""
from typing import List, Tuple

import torch

from neuralmonkey_b200.nn.projection import declare_multilayer_projection, multilayer_projection
from neuralmonkey_b200.params import zeros_initializer


class MultilayerPerceptron:
    def __init__(self, part, layer_configuration: List[int], dropout_keep_prob: float, output_size: int,
                 activation: str = "relu", name: str = "multilayer_perceptron") -> None:
        self.part = part
        self.layers = list(layer_configuration)
        self.dropout_keep_prob = dropout_keep_prob
        self.output_size = output_size
        self.activation = activation
        self.name = name

    def declare(self, in_size: int) -> None:
        last = declare_multilayer_projection(self.part, self.name + "/deep_output_mlp", in_size, self.layers)
        self.part.declare(self.name + "/classification_layer/kernel", [last, self.output_size])
        self.part.declare(self.name + "/classification_layer/bias", [self.output_size], zeros_initializer())

    def last_layer(self, mlp_input: torch.Tensor, train_mode: bool) -> torch.Tensor:
        """The input of the classification layer."""
        return multilayer_projection(self.part, mlp_input, self.name + "/deep_output_mlp", self.layers,
                                     self.activation, self.dropout_keep_prob, train_mode)

    @property
    def classification_layer(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(kernel [last, output_size], bias [output_size])."""
        return (self.part.var(self.name + "/classification_layer/kernel"),
                self.part.var(self.name + "/classification_layer/bias"))
