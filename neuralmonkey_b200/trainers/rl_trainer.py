"""Training objectives for reinforcement learning (reference: neuralmonkey/trainers/rl_trainer.py).

The sampling loops run under autograd (`Decoder.differentiable_loop` with `ops.sample_logits_step`); the rewards
come from an evaluator object over words, on the host, as in the reference."""
from typing import Callable, List

import numpy as np
import torch

from neuralmonkey_b200 import runtime
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.trainers.objective import Objective
from neuralmonkey_b200.trainers.self_critical_objective import batch_cached, check_rl_decoder, check_single_rank
from neuralmonkey_b200.vocabulary import END_TOKEN, PAD_TOKEN

# pylint: disable=invalid-name
RewardFunction = Callable[[np.ndarray, np.ndarray], np.ndarray]
# pylint: enable=invalid-name


class ReinforceObjective(Objective):
    # pylint: disable=too-many-arguments
    def __init__(self, decoder, reward_function: RewardFunction, subtract_baseline: bool = False,
                 normalize: bool = False, temperature: float = 1., ce_smoothing: float = 0., alpha: float = 1.,
                 sample_size: int = 1) -> None:
        """Objective for training with sentence-level feedback (rl_trainer.py:22-76).

        Depending on the options it is
        1) sample_size = 1, normalize = False, ce_smoothing = 0: the bandit objective (Eq. 2) of 'Bandit Structured
           Prediction for Neural Sequence-to-Sequence Learning' (http://www.aclweb.org/anthology/P17-1138);
           subtract_baseline = True is recommended;
        2) sample_size > 1, normalize = True, ce_smoothing = 0: Minimum Risk Training, 'Minimum Risk Training for
           Neural Machine Translation' (http://www.aclweb.org/anthology/P16-1159, Eq. 12);
        3) sample_size > 1, normalize = False, ce_smoothing = 0: the 'Reinforce' objective of 'Google's NMT System'
           (https://arxiv.org/pdf/1609.08144.pdf, Eq. 8);
        4) sample_size > 1, normalize = False, ce_smoothing > 0: its 'Mixed' objective (Eq. 9), ce_smoothing being
           its alpha.

        `alpha` sharpens the normalised distribution, `temperature` the sampling distribution.

        :param decoder: a recurrent decoder to sample from
        :param reward_function: any evaluator object: called as reward_function([hypothesis], [reference]) over
            words per sentence
        :param subtract_baseline: subtract the average reward of all samples seen so far
        :param normalize: re-normalise the probabilities of the samples
        :param sample_size: number of samples to obtain feedback for
        :param ce_smoothing: add the cross-entropy with this coefficient to the loss
        :param alpha: shape of the normalised distribution
        :param temperature: the softmax temperature for sampling
        """
        check_rl_decoder(decoder, "ReinforceObjective")
        if sample_size < 1:
            raise ValueError("sample_size must be at least 1")
        if temperature <= 0:
            raise ValueError("The softmax temperature must be positive")
        Objective.__init__(self, "{}_rl".format(decoder.name), decoder)
        self.reward_function = reward_function
        self.subtract_baseline = subtract_baseline
        self.normalize = normalize
        self.temperature = temperature
        self.ce_smoothing = ce_smoothing
        self.alpha = alpha
        self.sample_size = sample_size
        # the reference's reward_counter / reward_sum variables: float32, persistent across training steps and
        # not saved (its Saver skips reward_*)
        self.reward_counter = np.float32(0.0)
        self.reward_sum = np.float32(0.0)
    # pylint: enable=too-many-arguments

    graph_capturable = False

    @property
    def loss(self) -> torch.Tensor:
        return batch_cached(self, self._loss)

    def score_with_reward_function(self, references: np.ndarray, hypotheses: np.ndarray) -> np.ndarray:
        """Rewards [B] float32 of time-major id arrays (rl_trainer.py:83-115): each sentence is cut at the first
        </s> or <pad>, BPE pieces are joined ("@@ " removed) and the evaluator scores ([hypothesis], [reference])."""
        words = self.decoder.vocabulary.index_to_word
        rewards = []
        for refs, hyps in zip(references.transpose(), hypotheses.transpose()):
            seqs = []       # type: List[List[str]]
            for row in (refs, hyps):
                seq = []
                for token_id in row:
                    token = words[token_id]
                    if token in (END_TOKEN, PAD_TOKEN):
                        break
                    seq.append(token)
                seqs.append(" ".join(seq).replace("@@ ", "").split(" "))
            rewards.append(float(self.reward_function([seqs[1]], [seqs[0]])))
        return np.array(rewards, dtype=np.float32)

    def _loss(self) -> torch.Tensor:
        check_single_rank("ReinforceObjective")
        dec = self.decoder
        references = dec.train_inputs.cpu().numpy()
        rewards, logprobs = [], []
        for sample in range(self.sample_size):
            loop = dec.differentiable_loop(sample=True, temperature=self.temperature, sample_index=sample)
            rewards.append(self.score_with_reward_function(references, loop["symbols"].cpu().numpy()))
            nll, _ = dec.loop_nll(loop["states"], loop["symbols"], self.temperature)
            # no masking: otherwise shorter sentences are preferred (rl_trainer.py:138-140)
            logprobs.append(-nll.sum(0))
        rewards_stacked = np.stack(rewards)                # [sample_size, batch]
        if self.subtract_baseline:
            self.reward_counter = np.float32(self.reward_counter + np.float32(dec.batch_size * self.sample_size))
            self.reward_sum = np.float32(self.reward_sum + rewards_stacked.sum(dtype=np.float32))
            baseline = self.reward_sum / max(self.reward_counter, np.float32(1.0))
            rewards_stacked = rewards_stacked - baseline
        logprobs_stacked = torch.stack(logprobs)           # [sample_size, batch]
        if self.normalize:
            logprobs_stacked = torch.softmax(logprobs_stacked * self.alpha, dim=0)
        reward_t = runtime.to_device(torch.from_numpy(np.ascontiguousarray(rewards_stacked, dtype=np.float32)))
        batch_loss = (-reward_t * logprobs_stacked).sum(0).mean()
        if self.ce_smoothing > 0.0:
            batch_loss = batch_loss + self.ce_smoothing * dec.cost
        return batch_loss


def rl_objective(*args, **kwargs) -> ReinforceObjective:
    warn("Using deprecated rl_objective function. Use ReinforceObjective class directly.")
    return ReinforceObjective(*args, **kwargs)
