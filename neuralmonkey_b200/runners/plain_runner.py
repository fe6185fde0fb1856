"""PlainRunner (reference: neuralmonkey/runners/plain_runner.py): decodes `decoder.decoded` - the argmax
over logits[:, :, 1:] + 1 of the greedy loop, i.e. <pad> can never be produced - instead of the runner-side
argmax of GreedyRunner; a single session only."""
from typing import Callable, List, Optional, Union

from neuralmonkey_b200.decoders.autoregressive import AutoregressiveDecoder
from neuralmonkey_b200.decoders.ctc_decoder import CTCDecoder
from neuralmonkey_b200.runners.base_runner import BaseRunner
from neuralmonkey_b200.typecheck import check_argument_types

SupportedDecoder = Union[AutoregressiveDecoder, CTCDecoder]
Postprocessor = Optional[Callable[[List[List[str]]], List[List[str]]]]


class PlainRunner(BaseRunner):
    class Executable(BaseRunner.Executable):
        def execute(self) -> None:
            runner = self.executor
            decoder = runner.decoder
            decoded_tokens = decoder.vocabulary.vectors_to_sentences(decoder.decoded.cpu().numpy())
            if runner.postprocess is not None:
                decoded_tokens = runner.postprocess(decoded_tokens)
            losses = [0.0, 0.0]
            if self.compute_losses:
                losses = [float(decoder.train_loss), float(decoder.runtime_loss)]
            self.set_runner_result(outputs=decoded_tokens, losses=losses)

        def execute_sessions(self, activate, num_sessions: int) -> None:
            raise ValueError("PlainRunner needs exactly 1 execution result, got {}".format(num_sessions))

    def __init__(self, output_series: str, decoder: SupportedDecoder,
                 postprocess: Postprocessor = None) -> None:
        check_argument_types()
        BaseRunner.__init__(self, output_series, decoder)
        self.postprocess = postprocess

    @property
    def loss_names(self) -> List[str]:
        return ["train_loss", "runtime_loss"]
