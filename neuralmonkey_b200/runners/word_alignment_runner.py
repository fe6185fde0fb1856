"""WordAlignmentRunner (reference: neuralmonkey/runners/word_alignment_runner.py): the attention weights a decoder's
greedy run recorded on one of its attentions, per sentence as an [encoder states, run steps] matrix."""
from typing import List

from neuralmonkey_b200.attention.base_attention import BaseAttention
from neuralmonkey_b200.decoders.decoder import Decoder
from neuralmonkey_b200.runners.base_runner import BaseRunner, GraphExecutor
from neuralmonkey_b200.typecheck import check_argument_types


class WordAlignmentRunner(BaseRunner):

    class Executable(BaseRunner.Executable):
        def execute(self) -> None:
            runner = self.executor
            _ = runner.run_decoder.runtime_symbols      # the greedy run records the histories
            histories = runner.decoder.histories
            if runner.key not in histories:
                raise KeyError("Attention has no recorded histories under key '{}'".format(runner.key))
            alignment = histories[runner.key].permute(1, 2, 0).cpu().numpy()     # [batch, time, steps]
            self.set_runner_result(outputs=alignment, losses=[])

    def __init__(self, output_series: str, attention: BaseAttention, decoder: Decoder) -> None:
        check_argument_types()
        BaseRunner.__init__(self, output_series, attention)
        # the decoder runs the loop that records the attention: it is fed as well
        GraphExecutor.__init__(self, {attention, decoder})
        self.run_decoder = decoder
        self.key = "{}_run".format(decoder.name)

    @property
    def loss_names(self) -> List[str]:
        return []
