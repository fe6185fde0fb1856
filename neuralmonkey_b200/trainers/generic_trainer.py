"""Generic trainer (reference: neuralmonkey/trainers/generic_trainer.py:20-250).

One `train_step()` =
    zero the flat gradient buffer
    -> backward of the objectives (weight gradients accumulate straight into the arena)
    -> [data parallel: one all-reduce of gradients + loss sum + token count]
    -> nm_clip_adam_step: L1/L2 terms, per-tensor clip_by_norm, TF-Adam (K13)
with no device->host synchronisation inside; the losses are returned as device tensors.
"""
import math
import re
from collections.abc import Mapping
from typing import Any, Dict, List, Optional, Sequence

import torch

from neuralmonkey_b200 import distributed, lib, ops, runtime, tf
from neuralmonkey_b200.lib import call, ptr
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.model.feedable import Feedable
from neuralmonkey_b200.runners.base_runner import ExecutionResult, GraphExecutor
from neuralmonkey_b200.trainers.objective import Objective

BIAS_REGEX = re.compile(r"[Bb]ias")


class GenericTrainer(GraphExecutor, Feedable):
    @staticmethod
    def default_optimizer():
        return tf.AdamOptimizer(learning_rate=1e-4)

    # pylint: disable=too-many-arguments
    def __init__(self, objectives: Sequence[Objective], l1_weight: float = 0.0,
                 l2_weight: float = 0.0, clip_norm: float = None, optimizer=None,
                 var_scopes: List[str] = None, var_collection: str = None,
                 use_cuda_graph: bool = False) -> None:
        GraphExecutor.__init__(self, {obj.decoder for obj in objectives})
        # Capture zero-grad + forward + backward + clip/Adam of a batch shape once and replay it:
        # a step is ~700 kernel launches, i.e. ~7 ms of Python/driver time per step (`bench.py`
        # reports it as host_enqueue_ms_per_step) next to ~8 ms of GPU time.  Data parallel: two graphs
        # with the NCCL all-reduce between them.
        self.use_cuda_graph = use_cuda_graph
        self.capture_exchange = True     # data parallel: NCCL inside the step's graph (falls back if capture fails)
        self._graphs = {}   # shape key -> "seen" | "failed" | captured step
        self.MAX_GRAPHS = 4
        Feedable.__init__(self)
        self.objectives = objectives
        self.l1_weight = l1_weight
        self.l2_weight = l2_weight
        self.clip_norm = clip_norm
        self.var_scopes = var_scopes
        self.var_collection = var_collection
        self.optimizer = optimizer if optimizer is not None else self.default_optimizer()
        self.batches_per_update = 1
        if clip_norm is not None and clip_norm <= 0.0:
            raise ValueError("clip_norm must be positive")

    @property
    def global_step(self) -> int:
        """Shared by all trainers (several trainers alternate on one model in tests/bahdanau.ini): bias
        correction and learning-rate schedules follow the number of updates of the MODEL."""
        return runtime.global_step()

    @global_step.setter
    def global_step(self, value: int) -> None:
        runtime.set_global_step(value)

    @property
    def var_list(self) -> List[str]:
        """Names of the variables this trainer updates: all trainable ones, or with `var_scopes` those
        whose name starts with one of the scopes (tf.get_collection(collection, scope) matches the scope
        as a regular expression at the start of the name; generic_trainer.py:196-205)."""
        names = list(getattr(runtime.arena(), "train_names", []))
        if self.var_scopes is None:
            return names
        return [n for n in names if any(re.match(scope, n) for scope in self.var_scopes)]

    def _scope_restriction(self, base_flags: torch.Tensor):
        """(segment flags, gradient mask) that keep the variables outside `var_scopes` untouched: their
        gradients are zeroed and their segments flagged lazy-only, so the optimizer kernel skips every
        one of their elements (moments included) and adds no regularisation term to them.  (The reported
        L1 / L2 values then cover the trained variables only.)"""
        if not hasattr(self, "_scope_state"):
            arena = runtime.arena()
            included = set(self.var_list)
            keep = torch.tensor([1 if n in included else 0 for n in arena.train_names] or [0],
                                dtype=torch.uint8, device=base_flags.device)
            flags = torch.where(keep.bool(), base_flags, torch.full_like(base_flags, 2))
            lengths = (arena.seg_off[1:] - arena.seg_off[:-1]).to(keep.device)
            mask = torch.repeat_interleave(keep.to(torch.float32), lengths)
            self._scope_state = (flags, mask)
            self._excluded = [n for n in arena.train_names if n not in included]
        return self._scope_state

    # -- gradient exchange overlapped with the backward pass (K14) -------------------------------
    def _exchange_plan(self):
        """(encoder parts, early ranges, late ranges) of the flat gradient buffer.

        The variables of the parts DOWNSTREAM of the encoders (decoders, attentions: on the en-de model
        88 of 129 MB, on the Transformer 166 of 308 MB) have their final gradients as soon as the backward
        pass reaches the encoders, long before it ends - their all-reduce can run on NCCL's stream while
        the encoder is still being differentiated.  The buffer is sorted by variable name, so the
        variables of a part are contiguous; adjacent segments are merged into ranges."""
        if hasattr(self, "_plan"):
            return self._plan
        arena = runtime.arena()
        encoders, late_parts = [], set()
        for obj in self.objectives:
            for enc in getattr(obj.decoder, "encoders", None) or []:
                if enc not in encoders:
                    encoders.append(enc)
                if hasattr(enc, "get_dependencies"):
                    late_parts |= set(enc.get_dependencies()[1])
        late_names = {getattr(p, "name", None) for p in late_parts}
        early, late = [], []
        offs = [int(o) for o in arena.seg_off.tolist()]
        for i, name in enumerate(arena.train_names):
            target = late if name.split("/", 1)[0] in late_names else early
            lo, hi = offs[i], offs[i + 1]
            if target and target[-1][1] == lo:
                target[-1] = (target[-1][0], hi)
            else:
                target.append((lo, hi))
        if not encoders or not late or not early:
            early, late = [], [(0, arena.trainable_size)]
        self._plan = (encoders, early, late)
        return self._plan

    def _arm_early_exchange(self, works: list):
        """Evaluate the encoders first and hook their outputs: autograd runs the node with the highest
        sequence number among the ready ones, and every node of the decoders is now younger than every
        node of the encoders - so when the first gradient of an encoder output is complete, all decoder
        and attention gradients are final.  That moment starts the all-reduce of their ranges (async: NCCL's
        own stream, ordered after the kernels already issued; the backward pass goes on meanwhile)."""
        arena = runtime.arena()
        encoders, early, _late = self._exchange_plan()
        if not early:
            return
        tensors = []
        for enc in encoders:
            for attr in ("temporal_states", "spatial_states", "output"):
                try:
                    val = getattr(enc, attr)
                except (AttributeError, NotImplementedError, ValueError, TypeError):
                    continue
                if torch.is_tensor(val) and val.requires_grad and val.grad_fn is not None:
                    tensors.append(val)
        fired = []

        def hook(_grad):
            if not fired:
                fired.append(True)
                self.early_exchanges = getattr(self, "early_exchanges", 0) + 1
                # parameters used in plain torch expressions get their gradient in `.grad` (AccumulateGrad
                # nodes run before any older node): move those into the flat buffer before it is exchanged
                ops.join_weight_grads()            # the decoder-side weight gradients issued on the second stream
                arena.fold_autograd_grads()
                for lo, hi in early:
                    works.append(distributed.all_reduce_async(arena.grad_buffer[lo:hi]))
            return None

        for t in tensors:
            t.register_hook(hook)
        works.append(("armed", fired, early))

    def _finish_exchange(self, works: list) -> None:
        """All-reduce what the hook did not cover (the encoders' ranges and the statistic slots - or, when
        it never fired, everything) and make the compute stream wait for the exchange."""
        arena = runtime.arena()
        _enc, _early, late = self._exchange_plan()
        armed = [w for w in works if isinstance(w, tuple) and w[0] == "armed"]
        handles = [w for w in works if not isinstance(w, tuple)]
        tail = arena.trainable_size
        if armed and armed[0][1]:
            ranges = list(late)
            if ranges and ranges[-1][1] == tail:
                ranges[-1] = (ranges[-1][0], tail + arena.STAT_SLOTS)        # stats ride with the last range
            else:
                ranges.append((tail, tail + arena.STAT_SLOTS))
            for lo, hi in ranges:
                handles.append(distributed.all_reduce_async(arena.grad_buffer[lo:hi]))
        else:
            handles.append(distributed.all_reduce_async(arena.allreduce_view))
        timed = arena.params.is_cuda and not torch.cuda.is_current_stream_capturing()
        if timed:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        for h in handles:
            if h is not None:
                h.wait()
        if timed:       # how long the compute stream waited for the exchange after the backward pass was issued
            ev1.record()
            history = getattr(self, "_comm_history", None)
            if history is None:
                history = self._comm_history = []
            history.append([(ev0, ev1)])
            del history[:-8]
        del works[:]

    # -- one optimisation step ---------------------------------------------------------------
    def _backward(self, works: Optional[list] = None) -> Dict[str, torch.Tensor]:
        """Backward of the weighted objectives into the arena; fills the stat slots.
        Returns the device tensors reported as losses.  `works` (data parallel): a list that receives
        the handles of the gradient ranges whose all-reduce is started DURING the backward pass."""
        arena = runtime.arena()
        if works is not None:
            self._arm_early_exchange(works)
        exact = None
        if len(self.objectives) == 1 and self.objectives[0].gradients is None:
            exact = self.objectives[0].loss_sum_and_count
        if exact is not None:
            # token-mean loss: differentiate the SUM, divide by the (global) count in the
            # optimizer kernel -> N ranks reproduce the single-GPU token mean exactly
            loss_sum, count = exact
            w = self.objectives[0].weight
            ops.weight_grad_stream(arena.params.is_cuda)
            try:
                (loss_sum if w is None else loss_sum * w).backward()
            finally:
                ops.join_weight_grads()
                ops.weight_grad_stream(False)
            arena.fold_autograd_grads()
            arena.stats[0].copy_(loss_sum.detach())
            arena.stats[1].copy_(count.detach())
            return {"exact": True}
        total = None
        for obj in self.objectives:
            if obj.gradients is not None:
                raise NotImplementedError("objectives with explicit gradients (RL) are out of scope")
            w = 1.0 if obj.weight is None else obj.weight
            term = obj.loss * w
            total = term if total is None else total + term
        ops.weight_grad_stream(arena.params.is_cuda)
        try:
            total.backward()
        finally:
            ops.join_weight_grads()
            ops.weight_grad_stream(False)
        arena.fold_autograd_grads()
        return {"exact": False}

    # -- CUDA-graph replay of a whole step -------------------------------------------------------
    def _leaf_parts(self):
        return sorted((p for p in self.feedables if p is not self and hasattr(p, "static_inputs")),
                      key=lambda p: getattr(p, "name", type(p).__name__))

    def _graphed_step(self) -> Optional[Dict[str, Any]]:
        arena = runtime.arena()
        parts = self._leaf_parts()
        leaves = [(p, p.static_inputs()) for p in parts]
        key = tuple((getattr(p, "name", ""), k, tuple(t.shape), str(t.dtype), bool(p.train_mode), p.batch_size)
                    for p, d in leaves for k, t in sorted(d.items()))
        entry = self._graphs.get(key)
        if entry is None:
            self._graphs[key] = "seen"       # first batch of this shape: eager (it is the warm-up)
            return None
        if entry == "failed":
            return None
        if entry == "seen":
            captured = [k for k, v in self._graphs.items() if isinstance(v, tuple)]
            if len(captured) >= self.MAX_GRAPHS:          # bounded: a captured step owns its activations
                del self._graphs[captured[0]]
            if not hasattr(self, "_lr_dev"):
                self._lr_dev = torch.zeros(1, device=arena.params.device, dtype=torch.float32)
            static = [{k: t.clone() for k, t in d.items()} for _, d in leaves]
            try:
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                for p, st in zip(parts, static):
                    p.bind_static(st)
                graph2 = None
                if distributed.world_size() > 1 and self.capture_exchange:
                    # data parallel, everything in ONE graph: the ranges of the decoder side are
                    # all-reduced on NCCL's stream while the encoder is still being differentiated
                    # (the fork / join between the streams is captured as graph dependencies)
                    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                        arena.zero_grad()
                        works = []
                        self._backward(works)
                        self._finish_exchange(works)
                        self._adam_kernel(1.0, arena.stats[1:2], 0.0, self._lr_dev)
                elif distributed.world_size() > 1:
                    # the gradient exchange stays an eager NCCL call between two captured halves
                    # (backward | clip + Adam)
                    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                        arena.zero_grad()
                        self._backward()
                    graph2 = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph2, pool=graph.pool(), capture_error_mode="thread_local"):
                        self._adam_kernel(1.0, arena.stats[1:2], 0.0, self._lr_dev)
                else:
                    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                        arena.zero_grad()
                        self._backward()
                        self._adam_kernel(1.0, arena.stats[1:2], 0.0, self._lr_dev)
            except Exception as exc:  # pylint: disable=broad-except
                for p in parts:
                    p.reset_batch()
                if distributed.world_size() > 1 and self.capture_exchange:
                    warn("capturing the gradient exchange inside the step's CUDA graph failed ({}: {}); "
                         "falling back to two graphs around an eager all-reduce".format(type(exc).__name__, exc))
                    self.capture_exchange = False
                    torch.cuda.synchronize()
                    return None                     # this batch runs eagerly, the next one re-captures
                warn("CUDA-graph capture of the training step failed ({}: {}); staying eager".format(
                    type(exc).__name__, exc))
                self._graphs[key] = "failed"
                return None
            entry = self._graphs[key] = (graph, static, graph2)
            if distributed.world_size() > 1:
                distributed.register_cleanup(self._graphs.clear)   # graphs that captured NCCL go before NCCL does
        graph, static, graph2 = entry
        for (_, d), st in zip(leaves, static):
            for k, t in d.items():
                if st[k] is not t:
                    st[k].copy_(t)
        self._lr_dev.fill_(self._advance_step())
        graph.replay()
        if graph2 is not None:
            distributed.all_reduce_sum(arena.allreduce_view)
            graph2.replay()
        return {"losses": [arena.stats[0] / arena.stats[1]], "l1l2": self._l1l2}

    def train_step(self, apply_update: bool = True, grad_scale: float = 1.0,
                   zero_grad: bool = True) -> Dict[str, Any]:
        """Run one step on the batch currently fed to the model parts (train mode)."""
        arena = runtime.arena()
        if arena.params.is_cuda:
            runtime.advance_dropout()       # this step's dropout masks (read on the device: also by a replayed graph)
        if (self.use_cuda_graph and apply_update and zero_grad and grad_scale == 1.0
                and arena.params.is_cuda
                and len(self.objectives) == 1 and hasattr(type(self.objectives[0].decoder), "train_xent_sum")):
            out = self._graphed_step()
            if out is not None:
                return out
        if zero_grad:
            arena.zero_grad()
        world = distributed.world_size()
        works = [] if (world > 1 and apply_update) else None
        info = self._backward(works)
        losses = [obj.loss.detach() for obj in self.objectives]
        denominator = None
        if apply_update:
            if world > 1:
                if info["exact"] and grad_scale == 1.0:
                    lr_t = self._advance_step()
                    self._finish_exchange(works)
                    self._adam_kernel(1.0, arena.stats[1:2], lr_t, None)
                    return {"losses": [arena.stats[0] / arena.stats[1]], "l1l2": self._l1l2}
                self._finish_exchange(works)
            if info["exact"]:
                denominator = arena.stats[1:2]
                losses = [arena.stats[0] / arena.stats[1]]
            elif world > 1:
                grad_scale = grad_scale / world
            self.apply_gradients(grad_scale, denominator)
        return {"losses": losses, "l1l2": self._l1l2}

    @staticmethod
    def _waited_ms(waits) -> float:
        waits[-1][1].synchronize()
        return sum(float(a.elapsed_time(b)) for a, b in waits)

    @property
    def last_exposed_comm_ms(self) -> Optional[float]:
        """Device time the compute stream spent waiting for the gradient exchange after the backward pass was
        issued, in the last EAGERLY issued data-parallel step (None otherwise): what the overlap did not hide."""
        history = getattr(self, "_comm_history", None)
        if not history:
            return None
        return self._waited_ms(history[-1])

    @property
    def min_exposed_comm_ms(self) -> Optional[float]:
        """The smallest such time over the last (up to 8) eagerly issued steps.  An eagerly issued step is launched
        by the host kernel by kernel, so ranks drift apart by host jitter and the wait for the slowest rank lands
        in this figure; the minimum is the closest an eager step comes to the exchange alone."""
        history = getattr(self, "_comm_history", None)
        if not history:
            return None
        return min(self._waited_ms(w) for w in history)

    def _advance_step(self) -> float:
        """Increment the global step and the optimizer's own update count; returns Adam's bias-corrected step
        size.  The learning-rate schedule reads the GLOBAL step (shared by the trainers of an experiment,
        before its increment); the bias correction follows the number of updates THIS optimizer applied
        (TF's per-optimizer beta-power accumulators) - the two differ as soon as several trainers alternate."""
        opt = self.optimizer
        runtime.arena().optimizer_slot(opt)          # claims the slot (and a restored step count) on first use
        self.global_step += 1
        opt.steps += 1
        t = opt.steps
        lr = opt.lr_at(self.global_step - 1)
        return lr * math.sqrt(1.0 - opt.beta2 ** t) / (1.0 - opt.beta1 ** t)

    def apply_gradients(self, grad_scale: float = 1.0,
                        denominator: Optional[torch.Tensor] = None) -> None:
        self._adam_kernel(grad_scale, denominator, self._advance_step(), None)

    def _adam_kernel(self, grad_scale: float, denominator: Optional[torch.Tensor], lr_t: float,
                     lr_t_dev: Optional[torch.Tensor]) -> None:
        """Clip + regularise + Adam over the whole flat buffer."""
        arena = runtime.arena()
        opt = self.optimizer
        if not hasattr(self, "_l1l2_buf"):
            self._l1l2_buf = torch.zeros(2, device=arena.params.device, dtype=torch.float32)
        n = arena.trainable_size
        seg_flags = arena.seg_reg
        adam_m, adam_v = arena.optimizer_slot(opt)
        if getattr(opt, "lazy", False):
            # LazyAdam: embedding tables are updated only where a gradient arrived (flag bit 1)
            if not hasattr(self, "_lazy_flags"):
                lazy = torch.tensor([2 if ("embedding" in name) else 0 for name in arena.train_names] or [0],
                                    dtype=torch.uint8, device=arena.seg_reg.device)
                self._lazy_flags = arena.seg_reg | lazy
            seg_flags = self._lazy_flags
        if self.var_scopes is not None:
            seg_flags, mask = self._scope_restriction(seg_flags)
            arena.grads.mul_(mask)
        common = (float(opt.beta1), float(opt.beta2), float(opt.epsilon),
                  float(self.clip_norm) if self.clip_norm else 0.0, float(self.l1_weight), float(self.l2_weight))
        call("nm_clip_adam_step", ptr(arena.params), ptr(arena.grads), ptr(adam_m),
             ptr(adam_v), ptr(arena.seg_off), ptr(seg_flags), ptr(arena.seg_norms), n,
             len(arena.train_names), float(grad_scale), ptr(denominator), float(lr_t), *common,
             ptr(self._l1l2_buf), ptr(lr_t_dev), lib.stream())

    @property
    def _l1l2(self) -> torch.Tensor:
        return getattr(self, "_l1l2_buf", None)

    # -- executor protocol (runners/base_runner.py) --------------------------------------------
    def get_executable(self, compute_losses: bool = True, summaries: bool = True,
                       num_sessions: int = 1):
        if num_sessions != 1:
            raise ValueError("Trainer only supports execution in a single session")
        return _TrainExecutable(self)


class _TrainExecutable:
    def __init__(self, trainer: GenericTrainer) -> None:
        self.trainer = trainer
        self.result = None  # type: Optional[ExecutionResult]

    def execute(self) -> None:
        out = self.trainer.train_step()
        names = [obj.name for obj in self.trainer.objectives] + ["L1", "L2"]
        self.result = ExecutionResult(outputs={}, losses=_DeferredLosses(names, out["losses"], out["l1l2"]),
                                      size=self.trainer.objectives[0].decoder.batch_size,
                                      summaries=[])


class _DeferredLosses(Mapping):
    """{objective name: value, "L1": ..., "L2": ...} of one training step, read from the device when somebody
    LOOKS at it.  A step is issued asynchronously; converting its loss to a Python float right away would make the
    host wait for the device after every step, although the training loop only looks at the losses of the steps it
    logs (learning_utils.py) - so the host would prepare batch i+1 (padding, string -> index, upload) only after
    step i had finished instead of while it runs.  The tensors kept here are the step's own results (a replayed
    graph's loss is divided out of the statistic slots into a fresh tensor), so later steps do not change them."""

    def __init__(self, names, losses, l1l2) -> None:
        self._names = list(names)
        # the regularisation sums live in one buffer every step overwrites: keep this step's copy
        self._pending = (list(losses), l1l2.clone() if l1l2 is not None else None)
        self._values = None

    def _resolved(self):
        if self._values is None:
            losses, l1l2 = self._pending
            vals = [float(l) for l in losses]
            vals += [float(l1l2[0]), float(l1l2[1])] if l1l2 is not None else [0.0, 0.0]
            self._values = dict(zip(self._names, vals))
            self._pending = None
        return self._values

    def __getitem__(self, key):
        return self._resolved()[key]

    def __iter__(self):
        return iter(self._names)

    def __len__(self) -> int:
        return len(self._names)

    def __repr__(self) -> str:
        return repr(self._resolved())
