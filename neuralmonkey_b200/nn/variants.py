"""Model variants next to the hot path (SURVEY.md 8(f) N4): the Nematus GRU cell
(reference: neuralmonkey/nn/ortho_gru_cell.py:57-105) and the LSTM cell.

These variants are COMPOSED from operations whose kernels are parity-tested on the GPU (`ops.linear`,
`ops.gru_layer` with one step, `ops.bahdanau_attention`) plus ONE fused kernel per step for the gate
arithmetic (`ops.nematus_gru_gate`, `ops.lstm_gate`: nm_nematus_gate_*, nm_lstm_gate_*); they step through time instead of running the fused sequence kernels.  The oracle restates
them and is pinned to the reference's own code (tests/test_oracle_vs_reference_code.py);
tests/test_gpu_variants.py runs every one of them on the GPU against the oracle (on the exact engine at
1e-3 / 5e-5)."""
from typing import Tuple

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.params import block_orthogonal_initializer, zeros_initializer


class NematusGRUCell:
    """state' = u * state + (1 - u) * tanh(state_proj_c(state) * r + input_proj_c(x)),
    [r, u] = sigmoid(state_proj_g(state) + input_proj_g(x)): the reset gate is applied AFTER the state
    projection.  `use_state_bias` / `use_input_bias` as in the reference's constructor (:67-70)."""

    def __init__(self, part, scope: str, input_size: int, size: int, use_state_bias: bool = False,
                 use_input_bias: bool = True) -> None:
        self.part, self.scope, self.input_size, self.size = part, scope, input_size, size
        self.use_state_bias, self.use_input_bias = use_state_bias, use_input_bias

    def declare(self) -> None:
        for gate, width in (("gates", 2 * self.size), ("candidate", self.size)):
            pre = "{}/{}/".format(self.scope, gate)
            self.part.declare(pre + "input_proj/kernel", [self.input_size, width])
            if self.use_input_bias:
                self.part.declare(pre + "input_proj/bias", [width], zeros_initializer())
            self.part.declare(pre + "state_proj/kernel", [self.size, width], block_orthogonal_initializer())
            if self.use_state_bias:
                self.part.declare(pre + "state_proj/bias", [width], zeros_initializer())

    def _proj(self, gate: str, side: str, x: torch.Tensor, biased: bool) -> torch.Tensor:
        pre = "{}/{}/{}/".format(self.scope, gate, side)
        return ops.linear(x, self.part.var(pre + "kernel"), self.part.var(pre + "bias") if biased else None)

    def input_projections(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """The input halves for any number of leading dims (all time steps in one GEMM each)."""
        return (self._proj("gates", "input_proj", x, self.use_input_bias),
                self._proj("candidate", "input_proj", x, self.use_input_bias))

    def step(self, gates_in: torch.Tensor, cand_in: torch.Tensor, state: torch.Tensor) -> torch.Tensor:
        return ops.nematus_gru_gate(self._proj("gates", "state_proj", state, self.use_state_bias), gates_in,
                                    self._proj("candidate", "state_proj", state, self.use_state_bias), cand_in,
                                    state)

    def __call__(self, x: torch.Tensor, state: torch.Tensor) -> torch.Tensor:
        gates_in, cand_in = self.input_projections(x)
        return self.step(gates_in, cand_in, state)

    def sequence(self, x: torch.Tensor, lengths: torch.Tensor, reverse: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        """dynamic_rnn over [batch, time, input] with `sequence_length`: zero outputs and a carried state
        past each length; `reverse` walks every sentence backwards inside its length, which is what
        reverse_sequence -> dynamic_rnn -> reverse_sequence computes (recurrent.py:96-104)."""
        bsz, steps, _ = x.shape
        gates_in, cand_in = self.input_projections(x)
        state = torch.zeros(bsz, self.size, device=x.device, dtype=torch.float32)
        outputs = [None] * steps
        for t in (range(steps - 1, -1, -1) if reverse else range(steps)):
            live = (lengths > t).to(torch.float32).unsqueeze(1)
            new = self.step(gates_in[:, t], cand_in[:, t], state)
            outputs[t] = new * live
            state = new * live + state * (1.0 - live)
        return torch.stack(outputs, 1), state


class LSTMCell:
    """tf.nn.rnn_cell.LSTMCell with its defaults (what RNN_CELL_TYPES["LSTM"] builds: no peepholes, no
    projection, forget_bias = 1): [i, j, f, o] = [x, h] . kernel + bias; c' = sigmoid(f + 1) * c +
    sigmoid(i) * tanh(j); h' = sigmoid(o) * tanh(c')."""

    def __init__(self, part, scope: str, input_size: int, size: int) -> None:
        self.part, self.scope, self.input_size, self.size = part, scope, input_size, size

    def declare(self) -> None:
        self.part.declare(self.scope + "/kernel", [self.input_size + self.size, 4 * self.size])
        self.part.declare(self.scope + "/bias", [4 * self.size], zeros_initializer())

    def __call__(self, x: torch.Tensor, c: torch.Tensor, h: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        z = ops.linear(torch.cat([x, h], 1), self.part.var(self.scope + "/kernel"), self.part.var(self.scope + "/bias"))
        return ops.lstm_gate(z, c)

    def sequence(self, x: torch.Tensor, lengths: torch.Tensor, reverse: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        """dynamic_rnn semantics as NematusGRUCell.sequence; the final state handed on is h
        (encoders/recurrent.py:91-93,106-107)."""
        bsz, steps, _ = x.shape
        c = h = torch.zeros(bsz, self.size, device=x.device, dtype=torch.float32)
        outputs = [None] * steps
        for t in (range(steps - 1, -1, -1) if reverse else range(steps)):
            live = (lengths > t).to(torch.float32).unsqueeze(1)
            new_c, new_h = self(x[:, t], c, h)
            outputs[t] = new_h * live
            c, h = new_c * live + c * (1.0 - live), new_h * live + h * (1.0 - live)
        return torch.stack(outputs, 1), h
