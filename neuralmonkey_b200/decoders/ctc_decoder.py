"""Connectionist temporal classification head (reference: neuralmonkey/decoders/ctc_decoder.py:17-154).

Per frame of the encoder's states a distribution over the vocabulary plus a blank (the last class), trained with
the CTC loss and decoded greedily: tf.nn.ctc_loss / tf.nn.ctc_greedy_decoder there, the K16 kernels here
(`ops.ctc_loss`, `ops.ctc_greedy_decode`).  The projection is the 1x1 convolution of the reference, i.e. the
dense layer over the state axis, on the projection GEMM.  Activations are batch-major; `logits` is the
reference's time-major view of them.
"""
from typing import Any, Dict, List, Tuple

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import TemporalStateful
from neuralmonkey_b200.params import uniform_initializer, zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200.vocabulary import PAD_TOKEN_INDEX, Vocabulary, pad_batch


class CTCDecoder(ModelPart):
    """Connectionist Temporal Classification.

    See `tf.nn.ctc_loss`, `tf.nn.ctc_greedy_decoder` etc.
    """

    # pylint: disable=too-many-arguments
    def __init__(self,
                 name: str,
                 encoder: TemporalStateful,
                 vocabulary: Vocabulary,
                 data_id: str,
                 max_length: int = None,
                 merge_repeated_targets: bool = False,
                 merge_repeated_outputs: bool = True,
                 beam_width: int = 1,
                 reuse: ModelPart = None,
                 save_checkpoint: str = None,
                 load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        if beam_width > 1:
            raise NotImplementedError(
                "CTCDecoder '{}': beam_width={} needs tf.nn.ctc_beam_search_decoder, which is not restated here; "
                "only greedy decoding (beam_width=1) is available".format(name, beam_width))
        self.encoder = encoder
        self.vocabulary = vocabulary
        self.data_id = data_id
        self.max_length = max_length
        self.merge_repeated_targets = merge_repeated_targets
        self.merge_repeated_outputs = merge_repeated_outputs
        self.beam_width = beam_width
        self._target_tokens = None       # type: Any
        self._targets_host = None        # type: Any
    # pylint: enable=too-many-arguments

    def declare_variables(self) -> None:
        classes = len(self.vocabulary) + 1
        self.declare("state_to_word_W", [self.encoder.dimension, classes], uniform_initializer(-0.5, 0.5))
        self.declare("state_to_word_b", [classes], zeros_initializer())

    # -- feeding -------------------------------------------------------------------------------
    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: str}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, None]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        sentences = dataset.maybe_get_series(self.data_id)
        if sentences is None and train:
            raise ValueError("You must feed reference sentences when training")
        self._target_tokens = self._targets_host = None
        if sentences is not None:
            self._target_tokens = pad_batch(list(sentences), self.max_length)
            fd[self.data_id] = self._target_tokens
            rows = [[int(i) for i in ids if i != PAD_TOKEN_INDEX]
                    for ids in self.vocabulary.strings_to_indices(self._target_tokens).numpy()]
            width = len(self._target_tokens[0]) if self._target_tokens else 0
            self._targets_host = self._pack(rows, width)
            if self.merge_repeated_targets:     # TF's preprocess_collapse_repeated: only what the loss sees
                rows = [[s for i, s in enumerate(r) if i == 0 or s != r[i - 1]] for r in rows]
            labels, lengths = self._pack(rows, width)
            self.__dict__["_batch_cache"].update({"_labels": runtime.to_device(torch.from_numpy(labels)),
                                                  "_label_lengths": runtime.to_device(torch.from_numpy(lengths))})
        return fd

    @staticmethod
    def _pack(rows: List[List[int]], width: int) -> Tuple[np.ndarray, np.ndarray]:
        """Label rows as labels [B, width] int64 (zero-padded) and their lengths [B] int32."""
        labels = np.zeros((len(rows), width), dtype=np.int64)
        lengths = np.zeros(len(rows), dtype=np.int32)
        for row, kept in enumerate(rows):
            labels[row, :len(kept)] = kept
            lengths[row] = len(kept)
        return labels, lengths

    def static_inputs(self) -> Dict[str, Any]:
        if self._target_tokens is None:
            return {}
        return {"labels": self._labels, "label_lengths": self._label_lengths}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self.__dict__["_batch_cache"].update({"_labels": tensors["labels"],
                                                  "_label_lengths": tensors["label_lengths"]})

    # the labels the loss reads: the non-<pad> ids of every row, collapsed under merge_repeated_targets
    @tensor
    def _labels(self) -> torch.Tensor:
        raise ValueError("CTCDecoder '{}' has no reference series fed".format(self.name))

    @tensor
    def _label_lengths(self) -> torch.Tensor:
        raise ValueError("CTCDecoder '{}' has no reference series fed".format(self.name))

    # -- the reference's attributes ---------------------------------------------------------------
    @property
    def target_tokens(self) -> List[List[str]]:
        """The fed references padded by `pad_batch` ([batch, time] strings)."""
        return self._target_tokens

    @tensor
    def train_targets(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """The reference's sparse label tensor - the non-<pad> ids of every row, in order (`tf.where(params != PAD)`),
        repeats kept - as (labels [B, width of the padded batch] int64, lengths [B] int32)."""
        if self._targets_host is None:
            raise ValueError("CTCDecoder '{}' has no reference series fed".format(self.name))
        return tuple(runtime.to_device(torch.from_numpy(a)) for a in self._targets_host)

    @tensor
    def _logits_bm(self) -> torch.Tensor:
        """[batch, time, len(vocabulary) + 1]; the blank is the last class."""
        return ops.linear(self.encoder.temporal_states, self.var("state_to_word_W"), self.var("state_to_word_b"))

    @property
    def logits(self) -> torch.Tensor:
        """Time-major view [time, batch, classes] (ctc_decoder.py:121-150)."""
        return self._logits_bm.transpose(0, 1)

    @tensor
    def _loss_per_sentence(self) -> torch.Tensor:
        return ops.ctc_loss(self._logits_bm, self.encoder.lengths, self._labels, self._label_lengths,
                            self.merge_repeated_outputs)

    @tensor
    def cost(self) -> torch.Tensor:
        return self._loss_per_sentence.sum()

    @property
    def train_loss(self) -> torch.Tensor:
        return self.cost

    @property
    def runtime_loss(self) -> torch.Tensor:
        return self.cost

    @property
    def train_xent_sum(self) -> torch.Tensor:
        """The un-normalised training loss: a decoder that has one gets its training step captured in a CUDA graph
        (`GenericTrainer(use_cuda_graph=True)`)."""
        return self.cost

    @tensor
    def loss_sum_and_count(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(loss sum, count) for `CostObjective`: the trainers differentiate the sum and divide the gradient by the
        count on the device.  The CTC cost is a plain sum over the sentences, so the count is one."""
        return self.cost, torch.ones((), device=runtime.device(), dtype=torch.float32)

    @tensor
    def decoded(self) -> torch.Tensor:
        """Greedy CTC decoding, time-major [longest decoded sequence, batch] padded with </s>
        (sparse_tensor_to_dense(sparse_transpose(...), END_TOKEN_INDEX), ctc_decoder.py:73-88)."""
        ids, lengths = ops.ctc_greedy_decode(self._logits_bm, self.encoder.lengths, self.merge_repeated_outputs)
        longest = int(lengths.max()) if lengths.numel() else 0
        return ids[:, :longest].t()
