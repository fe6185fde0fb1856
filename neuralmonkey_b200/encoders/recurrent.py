"""Recurrent encoders (reference: neuralmonkey/encoders/recurrent.py:18-314).

`rnn_layer` runs a (bi)directional length-masked GRU over the whole sequence: the input
half of both GRUCell matmuls is one tensor-core GEMM over all B*T rows, the recurrence
is the K2 sequence kernel (`ops.gru_layer`).  The GRU cell is the one the five target configs use;
"NematusGRU" and "LSTM" (tests/small.ini, tests/nematus.ini) step through time with the cells of
`nn/variants.py` (SURVEY.md 8(f) N4; GPU-verified by tests/test_gpu_variants.py).
"""
from typing import List, NamedTuple, Tuple, Union

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import EmbeddedFactorSequence, EmbeddedSequence
from neuralmonkey_b200.model.stateful import TemporalStateful, TemporalStatefulWithOutput
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.nn.variants import LSTMCell, NematusGRUCell
from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200.params import (constant_initializer, ones_initializer,
                                      orthogonal_initializer, zeros_initializer)
from neuralmonkey_b200.vocabulary import Vocabulary

RNN_CELL_TYPES = ("NematusGRU", "GRU", "LSTM")
RNN_DIRECTIONS = ["forward", "backward", "bidirectional"]

RNNSpec = NamedTuple("RNNSpec", [("size", int), ("direction", str), ("cell_type", str)])
RNNSpecTuple = Union[Tuple[int], Tuple[int, str], Tuple[int, str, str]]


def _make_rnn_spec(size: int, direction: str = "bidirectional", cell_type: str = "GRU") -> RNNSpec:
    if size <= 0:
        raise ValueError("RNN size must be a positive integer. {} given.".format(size))
    if direction not in RNN_DIRECTIONS:
        raise ValueError("RNN direction must be one of {}. {} given."
                         .format(str(RNN_DIRECTIONS), direction))
    if cell_type not in RNN_CELL_TYPES:
        raise ValueError("RNN cell type must be one of {}. {} given."
                         .format(str(RNN_CELL_TYPES), cell_type))
    return RNNSpec(size, direction, cell_type)


def gru_cell_variables(part: ModelPart, scope: str, input_size: int, size: int) -> None:
    """Declare tf.contrib.rnn.GRUCell variables under `scope` with OrthoGRUCell's initialisers
    (nn/ortho_gru_cell.py:44-53): orthogonal kernels, gate bias 1, candidate bias 0."""
    part.declare(scope + "/gates/kernel", [input_size + size, 2 * size], orthogonal_initializer())
    part.declare(scope + "/gates/bias", [2 * size], constant_initializer(1.0))
    part.declare(scope + "/candidate/kernel", [input_size + size, size], orthogonal_initializer())
    part.declare(scope + "/candidate/bias", [size], zeros_initializer())


def gru_cell_tensors(part: ModelPart, scope: str):
    return (part.var(scope + "/gates/kernel"), part.var(scope + "/gates/bias"),
            part.var(scope + "/candidate/kernel"), part.var(scope + "/candidate/bias"))


class RecurrentEncoder(ModelPart, TemporalStatefulWithOutput):
    # pylint: disable=too-many-arguments
    def __init__(self, name: str, input_sequence: TemporalStateful, rnn_layers: List[RNNSpecTuple],
                 add_residual: bool = False, add_layer_norm: bool = False,
                 include_final_layer_norm: bool = True, dropout_keep_prob: float = 1.0,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.input_sequence = input_sequence
        self.dropout_keep_prob = dropout_keep_prob
        self.rnn_specs = [_make_rnn_spec(*r) for r in rnn_layers]
        self.add_residual = add_residual
        self.add_layer_norm = add_layer_norm
        self.include_final_layer_norm = include_final_layer_norm
        if self.dropout_keep_prob <= 0.0 or self.dropout_keep_prob > 1.0:
            raise ValueError("Dropout keep prob must be inside (0,1].")
        layer_sizes = [2 * layer.size if layer.direction == "bidirectional" else layer.size
                       for layer in self.rnn_specs]
        if add_residual and len(set(layer_sizes)) > 1:
            raise ValueError("When using residual connectiong, all layers must have the same "
                             "size, but are {}.".format(layer_sizes))
        self._layer_sizes = layer_sizes

    def _cell_scopes(self, i: int, spec: RNNSpec) -> List[str]:
        base = "rnn_{}_{}".format(i, spec.direction)
        # OrthoGRUCell passes its scope itself (nn/ortho_gru_cell.py:51); NematusGRUCell gets
        # TensorFlow's default layer name, the snake-cased class name
        cell = {"NematusGRU": "nematus_gru_cell", "LSTM": "lstm_cell", "GRU": "OrthoGRUCell"}[spec.cell_type]
        if spec.direction == "bidirectional":
            return [base + "/bidirectional_rnn/fw/" + cell, base + "/bidirectional_rnn/bw/" + cell]
        return [base + "/rnn/" + cell]

    def _variant_cell(self, spec: RNNSpec, scope: str, in_dim: int):
        cls = NematusGRUCell if spec.cell_type == "NematusGRU" else LSTMCell
        return cls(self, scope, in_dim, spec.size)

    def declare_variables(self) -> None:
        if hasattr(self.input_sequence, "ensure_declared"):
            self.input_sequence.ensure_declared()
        in_dim = self.input_sequence.dimension
        for i, spec in enumerate(self.rnn_specs):
            for scope in self._cell_scopes(i, spec):
                if spec.cell_type != "GRU":
                    self._variant_cell(spec, scope, in_dim).declare()
                else:
                    gru_cell_variables(self, scope, in_dim, spec.size)
            if self.add_layer_norm:
                self.declare("rnn_{}_{}/LayerNorm/gamma".format(i, spec.direction), [in_dim],
                             ones_initializer())
                self.declare("rnn_{}_{}/LayerNorm/beta".format(i, spec.direction), [in_dim],
                             zeros_initializer())
            in_dim = self._layer_sizes[i]
        if self.include_final_layer_norm:
            # both final layer_norm calls resolve to the SAME variables (recurrent.py:215-216)
            self.declare("LayerNorm/gamma", [in_dim], ones_initializer())
            self.declare("LayerNorm/beta", [in_dim], zeros_initializer())

    @property
    def dimension(self) -> int:
        return self._layer_sizes[-1]

    @tensor
    def rnn_input(self) -> torch.Tensor:
        return dropout(self.input_sequence.temporal_states, self.dropout_keep_prob, self.train_mode)

    def _rnn_layer(self, i: int, spec: RNNSpec, layer_input: torch.Tensor,
                   lengths: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """rnn_layer (recurrent.py:71-110)."""
        scopes = self._cell_scopes(i, spec)
        if spec.cell_type != "GRU":
            in_dim = layer_input.shape[-1]
            runs = [self._variant_cell(spec, scope, in_dim).sequence(layer_input, lengths, reverse)
                    for scope, reverse in zip(scopes, {"bidirectional": (False, True), "forward": (False,),
                                                       "backward": (True,)}[spec.direction])]
            return torch.cat([r[0] for r in runs], 2), torch.cat([r[1] for r in runs], 1)
        if spec.direction == "bidirectional":
            if hasattr(ops, "gru_bilayer") and lengths is not None:
                # both recurrences in one launch each way: the directions are independent
                out_fw, fin_fw, out_bw, fin_bw = ops.gru_bilayer(
                    layer_input, lengths, gru_cell_tensors(self, scopes[0]), gru_cell_tensors(self, scopes[1]))
                return torch.cat([out_fw, out_bw], 2), torch.cat([fin_fw, fin_bw], 1)
            out_fw, fin_fw, _ = ops.gru_layer(layer_input, *gru_cell_tensors(self, scopes[0]),
                                           lengths=lengths, reverse=False)
            out_bw, fin_bw, _ = ops.gru_layer(layer_input, *gru_cell_tensors(self, scopes[1]),
                                           lengths=lengths, reverse=True)
            return torch.cat([out_fw, out_bw], 2), torch.cat([fin_fw, fin_bw], 1)
        out, fin, _ = ops.gru_layer(layer_input, *gru_cell_tensors(self, scopes[0]), lengths=lengths,
                                    reverse=(spec.direction == "backward"))
        return out, fin

    @tensor
    def rnn(self) -> Tuple[torch.Tensor, torch.Tensor]:
        layer_input = self.rnn_input
        layer_final = layer_input[:, -1]
        lengths = self.input_sequence.lengths
        for i, spec in enumerate(self.rnn_specs):
            if self.add_layer_norm:
                pre = "rnn_{}_{}/LayerNorm/".format(i, spec.direction)
                layer_input = ops.layer_norm(layer_input, self.var(pre + "gamma"), self.var(pre + "beta"))
            layer_output, layer_final_output = self._rnn_layer(i, spec, layer_input, lengths)
            layer_output = dropout(layer_output, self.dropout_keep_prob, self.train_mode)
            layer_final_output = dropout(layer_final_output, self.dropout_keep_prob, self.train_mode)
            if self.add_residual and layer_input.shape[-1] == layer_output.shape[-1]:
                layer_input = layer_input + layer_output
                layer_final = layer_final + layer_final_output
            else:
                layer_input = layer_output
                layer_final = layer_final_output
        if self.include_final_layer_norm:
            gamma, beta = self.var("LayerNorm/gamma"), self.var("LayerNorm/beta")
            return (ops.layer_norm(layer_input, gamma, beta), ops.layer_norm(layer_final, gamma, beta))
        return layer_input, layer_final

    @tensor
    def temporal_states(self) -> torch.Tensor:
        return self.rnn[0]

    @tensor
    def temporal_mask(self) -> torch.Tensor:
        return self.input_sequence.temporal_mask

    @tensor
    def output(self) -> torch.Tensor:
        return self.rnn[1]


class SentenceEncoder(RecurrentEncoder):
    # pylint: disable=too-many-arguments,too-many-locals
    def __init__(self, name: str, vocabulary: Vocabulary, data_id: str, embedding_size: int,
                 rnn_size: int, rnn_cell: str = "GRU", rnn_direction: str = "bidirectional",
                 add_residual: bool = False, add_layer_norm: bool = False, max_input_len: int = None,
                 dropout_keep_prob: float = 1.0, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None,
                 embedding_initializer=None) -> None:
        """Embedded input sequence + one RNN layer (recurrent.py:236-314)."""
        check_argument_types()
        s_ckp = "input_{}".format(save_checkpoint) if save_checkpoint else None
        l_ckp = "input_{}".format(load_checkpoint) if load_checkpoint else None
        emb_initializers = None
        if embedding_initializer is not None:
            emb_initializers = [("embedding_matrix_0", embedding_initializer)]
        input_sequence = EmbeddedSequence(
            name="{}_input".format(name), vocabulary=vocabulary, data_id=data_id,
            embedding_size=embedding_size, max_length=max_input_len, save_checkpoint=s_ckp,
            load_checkpoint=l_ckp, initializers=emb_initializers)
        RecurrentEncoder.__init__(
            self, name=name, input_sequence=input_sequence,
            rnn_layers=[(rnn_size, rnn_direction, rnn_cell)], add_residual=add_residual,
            add_layer_norm=add_layer_norm, dropout_keep_prob=dropout_keep_prob, reuse=reuse,
            save_checkpoint=save_checkpoint, load_checkpoint=load_checkpoint,
            initializers=initializers)
        self.vocabulary = vocabulary
        self.data_id = data_id
        self.max_input_len = max_input_len


class FactoredEncoder(RecurrentEncoder):
    # pylint: disable=too-many-arguments,too-many-locals
    def __init__(self, name: str, vocabularies: List[Vocabulary], data_ids: List[str],
                 embedding_sizes: List[int], rnn_size: int, rnn_cell: str = "GRU",
                 rnn_direction: str = "bidirectional", add_residual: bool = False,
                 add_layer_norm: bool = False, max_input_len: int = None,
                 dropout_keep_prob: float = 1.0, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None,
                 input_initializers: InitializerSpecs = None) -> None:
        """Multi-factor input sequence + one RNN layer (recurrent.py:317-385)."""
        check_argument_types()
        s_ckp = "input_{}".format(save_checkpoint) if save_checkpoint else None
        l_ckp = "input_{}".format(load_checkpoint) if load_checkpoint else None
        input_sequence = EmbeddedFactorSequence(
            name="{}_input".format(name), vocabularies=vocabularies, data_ids=data_ids,
            embedding_sizes=embedding_sizes, max_length=max_input_len, save_checkpoint=s_ckp,
            load_checkpoint=l_ckp, initializers=input_initializers)
        RecurrentEncoder.__init__(
            self, name=name, input_sequence=input_sequence,
            rnn_layers=[(rnn_size, rnn_direction, rnn_cell)], add_residual=add_residual,
            add_layer_norm=add_layer_norm, dropout_keep_prob=dropout_keep_prob, reuse=reuse,
            save_checkpoint=save_checkpoint, load_checkpoint=load_checkpoint,
            initializers=initializers)
