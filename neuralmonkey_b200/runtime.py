"""Process-wide runtime context: the CUDA device this rank drives and the arena."""
import os
from typing import Optional

import torch

from neuralmonkey_b200.params import ParameterArena

_device = None  # type: Optional[torch.device]
_arena = None  # type: Optional[ParameterArena]
_global_step = 0   # tf.train.get_or_create_global_step(): ONE counter shared by every trainer of the experiment


def device() -> torch.device:
    """cuda:LOCAL_RANK.  There is no CPU execution path: model tensors live on the GPU."""
    global _device
    if _device is None:
        if not torch.cuda.is_available():
            raise RuntimeError(
                "neuralmonkey_b200 needs a CUDA device (sm_90a, H100); no CPU fallback exists")
        local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local_rank)
        _device = torch.device("cuda", local_rank)
    return _device


def arena() -> ParameterArena:
    """The arena model parts declare their variables in (one per experiment)."""
    global _arena
    if _arena is None:
        _arena = ParameterArena()
    return _arena


def reset() -> None:
    """Start a fresh experiment (new arena, global step 0)."""
    global _arena, _global_step, _dropout_state, _dropout_site
    _arena = None
    _global_step = 0
    _dropout_state = None
    _dropout_site = 0


# -- dropout random stream (kernel-side Philox: csrc/dropout.cu) ------------------------------------------
_dropout_state = None  # type: Optional[torch.Tensor]   # device int64 {seed, step}
_dropout_site = 0      # dropout calls since the last advance, in program order


def dropout_state() -> torch.Tensor:
    """Device {seed, step} the dropout kernels read.  The seed is torch's (the experiment's `random_seed`)."""
    global _dropout_state
    if _dropout_state is None:
        _dropout_state = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64,
                                      device=device())
    return _dropout_state


def advance_dropout() -> None:
    """New masks from here on: once per training step, BEFORE the step is issued or replayed (the increment is
    a device operation outside the step's CUDA graph, which reads `step` when it runs)."""
    global _dropout_site
    dropout_state()[1:2].add_(1)
    _dropout_site = 0


def next_dropout_site() -> int:
    """Number of this dropout call within the step (a captured step replays the numbers it was captured with)."""
    global _dropout_site
    _dropout_site += 1
    return _dropout_site


def global_step() -> int:
    """The experiment's global step (reference: generic_trainer.py:193-195 - every trainer's train_op
    increments the same tf global_step variable, which the learning-rate schedules read and the Saver stores)."""
    return _global_step


def set_global_step(value: int) -> None:
    global _global_step
    _global_step = int(value)


def to_device(host: torch.Tensor) -> torch.Tensor:
    """Host tensor -> device without stalling the host.  A copy from pageable memory waits for
    everything queued on the stream before it (the next step's feed would serialise with the
    previous step's kernels); staging through the pinned-memory allocator keeps it asynchronous."""
    dev = device()
    if host.is_cuda or dev.type != "cuda":
        return host.to(dev)
    if not host.is_pinned():
        host = host.contiguous().pin_memory()
    return host.to(dev, non_blocking=True)
