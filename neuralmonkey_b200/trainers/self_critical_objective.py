"""Self-critical training objective (reference: neuralmonkey/trainers/self_critical_objective.py).

Self-critical learning is a modification of REINFORCE that uses the reward of the train-time decoder output as the
baseline of the update (https://arxiv.org/pdf/1612.00563.pdf).  The scored hypothesis comes from the greedy loop run
under autograd (`Decoder.differentiable_loop`); the rewards of the two index-based metrics here are computed on the
device (`ops.sentence_ngram_reward`)."""
from typing import Callable, Optional

import numpy as np
import torch

from neuralmonkey_b200 import distributed, ops, runtime
from neuralmonkey_b200.trainers.objective import Objective

# pylint: disable=invalid-name
RewardFunction = Callable[[np.ndarray, np.ndarray], np.ndarray]
# pylint: enable=invalid-name


def check_rl_decoder(decoder, objective: str) -> None:
    """The objectives differentiate the loop of a recurrent `Decoder` (the reference types them
    `Objective[Decoder]`)."""
    from neuralmonkey_b200.decoders.decoder import Decoder
    if not isinstance(decoder, Decoder):
        raise TypeError("{} needs a recurrent decoders.decoder.Decoder, got {}".format(objective,
                                                                                     type(decoder).__name__))


def check_single_rank(objective: str) -> None:
    if distributed.world_size() > 1:
        raise RuntimeError("{} runs on one rank only: its rewards and baseline are per-process state and its loss "
                           "is not split into a sum and a count the data-parallel ranks could combine"
                           .format(objective))


def batch_cached(objective: Objective, compute: Callable[[], torch.Tensor]) -> torch.Tensor:
    """The loss of the batch currently fed to the objective's decoder, computed once: it is read again after the
    backward pass, which must neither sample nor update a baseline a second time."""
    cache = objective.decoder.__dict__.setdefault("_batch_cache", {})
    key = ("objective_loss", id(objective))
    if key not in cache:
        cache[key] = compute()
    return cache[key]


def score_rewards(reward_function, references: torch.Tensor, hypotheses: torch.Tensor) -> torch.Tensor:
    """[B] float32 device rewards of time-major id tensors.  `sentence_bleu` / `sentence_gleu` run on the device;
    any other callable gets host numpy [T, B] arrays, as tf.py_func hands them over, and returns [B] float32."""
    if getattr(reward_function, "takes_device_tensors", False):
        return reward_function(references, hypotheses)
    out = reward_function(references.cpu().numpy(), hypotheses.cpu().numpy())
    out = np.asarray(out)
    if out.dtype != np.float32 or out.shape != (references.shape[1],):
        raise ValueError("a reward function must return [batch] float32, got {} {}".format(out.dtype, out.shape))
    return runtime.to_device(torch.from_numpy(out))


class SelfCriticalObjective(Objective):
    """Self-critical objective.

    Baseline: the reward of the argmax of the teacher-forced logits (the pass `decoder.cost` comes from).  Scored:
    the reward of the unmasked argmax of the greedy loop.  Loss, as the reference writes it:

        -sum((r_greedy - r_train) * NLL(greedy argmax) * runtime_mask) / sum(runtime_mask)

    (0 when every row finished at the first step, where the reference's 0 / 0 gives NaN.)

    This sign is the opposite of Rennie et al.'s (their gradient increases the likelihood of hypotheses that beat
    the baseline; minimising this loss lowers it).  It is ported as written: parity with the reference is what
    this package keeps, and changing it changes what existing configurations train.
    """

    def __init__(self, decoder, reward_function: RewardFunction, weight: float = None) -> None:
        check_rl_decoder(decoder, "SelfCriticalObjective")
        Objective.__init__(self, "{}_self_critical".format(decoder.name), decoder)
        self.reward_function = reward_function
        self._weight = weight

    graph_capturable = False

    @property
    def weight(self) -> Optional[float]:
        return self._weight

    @property
    def loss(self) -> torch.Tensor:
        return batch_cached(self, self._loss)

    def _loss(self) -> torch.Tensor:
        check_single_rank("SelfCriticalObjective")
        dec = self.decoder
        train_decoded = dec._train_xent_result[2].t()          # [T, B] argmax of the teacher-forced logits
        loop = dec.differentiable_loop(sample=False)
        runtime_decoded = loop["argmax"]
        reference = dec.train_inputs
        with torch.no_grad():
            train_reward = score_rewards(self.reward_function, reference, train_decoded)
            runtime_reward = score_rewards(self.reward_function, reference, runtime_decoded)
        nll, _ = dec.loop_nll(loop["states"], runtime_decoded)
        mask = loop["mask"].to(torch.float32)
        score = reinforce_score(runtime_reward, train_reward, runtime_decoded, nll)
        # every row finishing at the first step leaves no unmasked position: the reference divides 0 by 0 there
        # and its NaN loss poisons every parameter through the update; the loss is 0 here
        return -(score * mask).sum() / mask.sum().clamp_min(1.0)


def reinforce_score(reward: torch.Tensor, baseline: torch.Tensor, decoded: torch.Tensor,
                    logits: torch.Tensor) -> torch.Tensor:
    """Cost whose derivative is the REINFORCE equation (self_critical_objective.py:95-121): the negative
    log-likelihood of the decoded symbols [T, B] times the reward difference, which is a constant.

    The reference passes the logits [T, B, V] and takes the NLL of `decoded` from them.  Here the vocabulary
    projection and its softmax stay in one fused kernel, so `logits` is what that kernel returns for `decoded`:
    their per-position NLL [T, B] (`Decoder.loop_nll`)."""
    if logits.shape != decoded.shape:
        raise ValueError("reinforce_score takes the NLL [time, batch] of the decoded symbols (Decoder.loop_nll), "
                         "got {} for symbols {}".format(tuple(logits.shape), tuple(decoded.shape)))
    return (reward - baseline).detach().unsqueeze(0) * logits


def sentence_bleu(references, hypotheses) -> torch.Tensor:
    """Index-based sentence-level BLEU (self_critical_objective.py:124-162), on the device: whatever the decoder
    uses as a unit is a token.  references [T_r, B], hypotheses [T_h, B] int64 ids (tensors or arrays); returns
    [B] float32 on the device."""
    return _device_reward(references, hypotheses, "bleu")


def sentence_gleu(references, hypotheses) -> torch.Tensor:
    """Index-based sentence GLEU (self_critical_objective.py:165-200): min of precision and recall over 1..4-grams.
    Where the reference divides 0 by 0 (no hypothesis or no reference n-gram) its assert fails; the score is 0.0
    here."""
    return _device_reward(references, hypotheses, "gleu")


sentence_bleu.takes_device_tensors = True
sentence_gleu.takes_device_tensors = True


def _device_reward(references, hypotheses, mode: str) -> torch.Tensor:
    def dev(x):
        x = torch.as_tensor(x, dtype=torch.int64)
        return x if x.is_cuda else runtime.to_device(x)
    return ops.sentence_ngram_reward(dev(references), dev(hypotheses), mode)

