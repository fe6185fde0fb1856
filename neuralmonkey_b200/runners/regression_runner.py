"""RegressionRunner (reference: neuralmonkey/runners/regression_runner.py): the predictions of a
`SequenceRegressor` ([batch, dimension] as lists), averaged over the sessions of an ensemble, with the cost summed
over them as the loss "mse"."""
from typing import Callable, List

import numpy as np

from neuralmonkey_b200.decoders.sequence_regressor import SequenceRegressor
from neuralmonkey_b200.runners.base_runner import BaseRunner
from neuralmonkey_b200.typecheck import check_argument_types

# pylint: disable=invalid-name
Postprocessor = Callable[[List[float]], List[float]]
# pylint: enable=invalid-name


class RegressionRunner(BaseRunner):
    """A runnner that takes the predictions of a sequence regressor."""

    class Executable(BaseRunner.Executable):
        def _session_result(self) -> dict:
            decoder = self.executor.decoder
            result = {"prediction": decoder.predictions.detach().cpu().numpy()}
            if decoder._targets is not None:     # pylint: disable=protected-access
                result["mse"] = float(decoder.cost)
            return result

        def execute(self) -> None:
            self.collect_results([self._session_result()])

        def execute_sessions(self, activate, num_sessions: int) -> None:
            results = []
            for index in range(num_sessions):
                activate(index)
                results.append(self._session_result())
            self.collect_results(results)

        def collect_results(self, results: List[dict]) -> None:
            predictions_sum = np.zeros_like(results[0]["prediction"])
            mse_loss = 0.
            for sess_result in results:
                if "mse" in sess_result:
                    mse_loss += sess_result["mse"]
                predictions_sum += sess_result["prediction"]
            predictions = (predictions_sum / len(results)).tolist()
            if self.executor.postprocess is not None:
                predictions = self.executor.postprocess(predictions)
            self.set_runner_result(outputs=predictions, losses=[mse_loss])

    def __init__(self, output_series: str, decoder: SequenceRegressor, postprocess: Postprocessor = None) -> None:
        check_argument_types()
        BaseRunner.__init__(self, output_series, decoder)
        self.postprocess = postprocess

    @property
    def loss_names(self) -> List[str]:
        return ["mse"]
