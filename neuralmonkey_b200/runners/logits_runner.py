"""LogitsRunner (reference: neuralmonkey/runners/logits_runner.py): the decoder's `decoded_logits` [time, batch,
classes], or their softmax, as text: per sentence the steps' values comma-joined (`str()` of numpy float32) and the
steps tab-joined, or the single value at `pick_index`.  As in the reference, a `pick_index` of 0 is treated as
unset.  Formatting happens on the host from the float32 logits, exactly as the reference does it."""
from typing import List, Optional

import numpy as np

from neuralmonkey_b200.runners.base_runner import BaseRunner
from neuralmonkey_b200.typecheck import check_argument_types


class LogitsRunner(BaseRunner):
    """A runner which takes the output from decoder.decoded_logits."""

    class Executable(BaseRunner.Executable):
        def execute(self) -> None:
            decoder = self.executor.decoder
            train_loss = runtime_loss = 0.0
            if self.compute_losses:
                train_loss = float(decoder.train_loss)
                runtime_loss = float(decoder.runtime_loss)
            self.collect_results([{"logits": decoder.decoded_logits.detach().cpu().numpy(),
                                   "train_loss": train_loss, "runtime_loss": runtime_loss}])

        def execute_sessions(self, activate, num_sessions: int) -> None:
            raise ValueError("LogitsRunner needs exactly 1 execution result, got {}".format(num_sessions))

        def collect_results(self, results: List[dict]) -> None:
            if len(results) != 1:
                raise ValueError("LogitsRunner needs exactly 1 execution result, got {}".format(len(results)))
            train_loss = results[0]["train_loss"]
            runtime_loss = results[0]["runtime_loss"]
            logits_list = results[0]["logits"]      # (time, batch, classes)
            outputs = [[] for _ in logits_list[0]]  # type: List[List[str]]
            for time_step in logits_list:
                for logits, output_list in zip(time_step, outputs):
                    if self.executor.normalize:
                        logits = np.exp(logits) / np.sum(np.exp(logits), axis=0)
                    if self.executor.pick_index:
                        instance_logits = str(logits[self.executor.pick_index])
                    else:
                        instance_logits = ",".join(str(l) for l in logits)
                    output_list.append(instance_logits)
            str_outputs = [["\t".join(l)] for l in outputs]
            self.set_runner_result(outputs=str_outputs, losses=[train_loss, runtime_loss])

    def __init__(self, output_series: str, decoder, normalize: bool = True, pick_index: int = None,
                 pick_value: str = None) -> None:
        check_argument_types()
        BaseRunner.__init__(self, output_series, decoder)
        if pick_index is not None and pick_value is not None:
            raise ValueError("Either a pick index or a vocabulary value can be specified, not both at the same "
                             "time.")
        self.pick_index = None  # type: Optional[int]
        self.normalize = normalize
        if pick_value is not None:
            if pick_value in self.decoder.vocabulary:
                self.pick_index = self.decoder.vocabulary.index_to_word.index(pick_value)
            else:
                raise ValueError("Value '{}' is not in vocabulary of decoder '{}'".format(pick_value, decoder.name))
        else:
            self.pick_index = pick_index

    @property
    def loss_names(self) -> List[str]:
        return ["train_loss", "runtime_loss"]
