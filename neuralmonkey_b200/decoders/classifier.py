"""A multilayer-perceptron classifier over encoder outputs (reference: neuralmonkey/decoders/classifier.py).

The API pretends it is an RNN decoder that always generates a sequence of length exactly one, so the existing
`GreedyRunner` decodes it: `decoded`, `decoded_logits`, `runtime_logprobs` and `runtime_argmax` are [1, batch, ...].
The classification layer and its cross-entropy are one `ops.logits_xent` call (no <unk> suppression,
unk_index = -1), which also gives the first-index argmax and the logsumexp the log-probabilities are taken from.
Kernel and bias of the layer sit side by side in the parameter arena, so in training that call runs on the fp16
wgmma vocabulary kernels (fp32 accumulation); `decoded_logits` are the logits that engine computes."""
from typing import Any, Dict, List, Tuple

import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decoders.encoder_projection import _encoder_output_size
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import Stateful
from neuralmonkey_b200.nn.mlp import MultilayerPerceptron
from neuralmonkey_b200.nn.projection import activation_name
from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200.vocabulary import Vocabulary, pad_batch


class Classifier(ModelPart):
    """A simple MLP classifier over encoders."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, encoders: List[Stateful], vocabulary: Vocabulary, data_id: str,
                 layers: List[int], activation_fn: str = "relu", dropout_keep_prob: float = 0.5,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.encoders = encoders
        self.vocabulary = vocabulary
        self.data_id = data_id
        self.layers = layers
        self.activation_fn = activation_name(activation_fn)
        self.dropout_keep_prob = dropout_keep_prob
        self.max_output_len = 1
        self.mlp = MultilayerPerceptron(self, layers, dropout_keep_prob, len(vocabulary), self.activation_fn)
        self._labels = None  # type: Any
    # pylint: enable=too-many-arguments

    def declare_variables(self) -> None:
        self.mlp.declare(sum(_encoder_output_size(enc) for enc in self.encoders))

    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: str}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        sentences = dataset.maybe_get_series(self.data_id)
        self._labels = None
        if sentences is not None:
            labels = [l[0] for l in pad_batch(list(sentences), self.max_output_len)]
            fd[self.data_id] = labels
            self._labels = runtime.to_device(self.vocabulary.strings_to_indices([labels])[0])
        return fd

    def static_inputs(self) -> Dict[str, Any]:
        return {"labels": self._labels} if self._labels is not None else {}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self._labels = tensors["labels"]

    @tensor
    def gt_inputs(self) -> torch.Tensor:
        """The fed labels as vocabulary indices [batch] int64."""
        if self._labels is None:
            raise ValueError("Classifier '{}' has no labels fed".format(self.name))
        return self._labels

    @tensor
    def _mlp_input(self) -> torch.Tensor:
        outputs = [enc.output for enc in self.encoders]
        return outputs[0] if len(outputs) == 1 else torch.cat(outputs, 1)

    @tensor
    def _classification(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """(xent [B], lse [B], argmax [B], logits [B, classes]).  Without labels the cross-entropy is zero."""
        x = self.mlp.last_layer(self._mlp_input, self.train_mode)
        kernel, bias = self.mlp.classification_layer
        rows = x.shape[0]
        if self._labels is not None:
            targets = self._labels
            weights = torch.ones(rows, device=x.device, dtype=torch.float32)
        else:
            targets = torch.zeros(rows, device=x.device, dtype=torch.int64)
            weights = torch.zeros(rows, device=x.device, dtype=torch.float32)
        return ops.logits_xent(x, kernel, bias, targets, weights, unk_index=-1, keep_logits=True)

    @tensor
    def _xent_sum(self) -> torch.Tensor:
        self.gt_inputs      # pylint: disable=pointless-statement  (raises without labels)
        return self._classification[0].sum()

    @tensor
    def loss_with_gt_ins(self) -> torch.Tensor:
        """Mean cross-entropy over the batch."""
        return self._xent_sum / self._classification[0].shape[0]

    @property
    def loss_with_decoded_ins(self) -> torch.Tensor:
        return self.loss_with_gt_ins

    @property
    def cost(self) -> torch.Tensor:
        return self.loss_with_gt_ins

    @property
    def train_loss(self) -> torch.Tensor:
        return self.loss_with_gt_ins

    @property
    def runtime_loss(self) -> torch.Tensor:
        return self.loss_with_decoded_ins

    @tensor
    def loss_sum_and_count(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(cross-entropy sum, batch size) for `CostObjective`: the trainers differentiate the sum and divide by the
        count on the device, so data-parallel ranks reproduce the single-GPU batch mean."""
        count = torch.full((), float(self._classification[0].shape[0]), device=runtime.device(), dtype=torch.float32)
        return self._xent_sum, count

    @tensor
    def decoded_seq(self) -> torch.Tensor:
        """[1, batch] int64: the first-index argmax of the logits."""
        return self._classification[2].unsqueeze(0)

    @property
    def decoded(self) -> torch.Tensor:
        return self.decoded_seq

    @property
    def runtime_argmax(self) -> torch.Tensor:
        return self.decoded_seq

    @tensor
    def decoded_logits(self) -> torch.Tensor:
        """[1, batch, classes]."""
        return self._classification[3].unsqueeze(0)

    @tensor
    def runtime_logprobs(self) -> torch.Tensor:
        """[1, batch, classes]: log_softmax of the logits."""
        _, lse, _, logits = self._classification
        return ops.log_softmax_from_lse(logits, lse).unsqueeze(0)
