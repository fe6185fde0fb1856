"""A multilayer-perceptron regression over encoder outputs (reference:
neuralmonkey/decoders/sequence_regressor.py).  The cost is mean((predictions [B, dimension] - target[:, None])^2)
on the K18 squared-error kernels (`ops.squared_error`); the target of a sentence is the first value of its float
vector."""
from typing import Any, Dict, List

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decoders.encoder_projection import _encoder_output_size
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import Stateful
from neuralmonkey_b200.nn.projection import activation_name, declare_multilayer_projection, multilayer_projection
from neuralmonkey_b200.params import zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types


class SequenceRegressor(ModelPart):
    """A simple MLP regression over encoders."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, encoders: List[Stateful], data_id: str, layers: List[int] = None,
                 activation_fn: str = "relu", dropout_keep_prob: float = 1.0, dimension: int = 1,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.encoders = encoders
        self.data_id = data_id
        self.max_output_len = 1
        self.dimension = dimension
        self._layers = list(layers) if layers is not None else []
        self._activation_fn = activation_name(activation_fn)
        self._dropout_keep_prob = dropout_keep_prob
        self._targets = None  # type: Any
    # pylint: enable=too-many-arguments

    def declare_variables(self) -> None:
        width = declare_multilayer_projection(self, "mlp", sum(_encoder_output_size(e) for e in self.encoders),
                                              self._layers)
        self.declare("output_projection/kernel", [width, self.dimension])
        self.declare("output_projection/bias", [self.dimension], zeros_initializer())

    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: float}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        series = dataset.maybe_get_series(self.data_id)
        self._targets = None
        if series is not None:
            firsts = list(zip(*list(series)))[0]
            fd[self.data_id] = firsts
            self._targets = runtime.to_device(torch.from_numpy(np.asarray(firsts, dtype=np.float32)))
        return fd

    def static_inputs(self) -> Dict[str, Any]:
        return {"targets": self._targets} if self._targets is not None else {}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self._targets = tensors["targets"]

    @tensor
    def train_inputs(self) -> torch.Tensor:
        """The fed targets [batch] float32."""
        if self._targets is None:
            raise ValueError("SequenceRegressor '{}' has no targets fed".format(self.name))
        return self._targets

    @tensor
    def _mlp_input(self) -> torch.Tensor:
        outputs = [enc.output for enc in self.encoders]
        return outputs[0] if len(outputs) == 1 else torch.cat(outputs, 1)

    @tensor
    def predictions(self) -> torch.Tensor:
        """[batch, dimension]."""
        hidden = multilayer_projection(self, self._mlp_input, "mlp", self._layers, self._activation_fn,
                                       self._dropout_keep_prob, self.train_mode)
        return ops.linear(hidden, self.var("output_projection/kernel"), self.var("output_projection/bias"))

    @tensor
    def cost(self) -> torch.Tensor:
        return ops.squared_error(self.predictions, self.train_inputs)

    @property
    def train_loss(self) -> torch.Tensor:
        return self.cost

    @property
    def runtime_loss(self) -> torch.Tensor:
        return self.cost

    @property
    def decoded(self) -> torch.Tensor:
        return self.predictions
