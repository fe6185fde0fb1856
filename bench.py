#!/usr/bin/env python3
"""Benchmark of the hot path BASELINE.json names.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--workload ende|transformer]

Default workload (the configuration BASELINE.json's metric is quoted on): training throughput of the
Bahdanau en-de model (examples/translation.ini dims: E = He = H = O = 300, C = A = 600, Tx = Ty = 50,
batch 256 per GPU, synthetic V = 32000) in non-pad target tokens per second over full optimizer steps
(forward + backward + [gradient exchange] + clip + Adam).  `--workload transformer` runs the 1->8 GPU
configuration BASELINE.json names for scaling (tests/transformer.ini at L=6 d=512, 4096 target tokens per
GPU and step, LazyAdam + Noam) with the same contract.

One JSON line on stdout (rank 0).  `value` is device-resident throughput (ids already in HBM); `e2e` feeds
every step from pinned host memory and reads the loss back.  `roofline` describes the dominant kernel
(timed with CUDA events inside eagerly issued steps), `cpu_baseline` times the CPU oracle restatement of the
same step on a bounded sample, `parity` compares the benched engine's loss with the oracle's on that
sample.  At N=1 the other configurations of BASELINE.json (RNN greedy / beam-8 decoding, Transformer
training, Transformer beam-8 decoding, VGG captioning) are measured the same way under `extra_workloads`,
each with its own roofline / cpu_baseline / e2e objects (bench_workloads.py).

`--impl reference` runs ONLY the CPU restatement (the reference's TF-1.12 path cannot run here:
SURVEY.md 8(c)) on the workload's shape, all host threads, a bounded number of sentences per step.
The models are built from INI text through the package's configuration builder (bench_models.py).
"""
import argparse
import contextlib
import json
import os
import re
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

METRIC = "train_target_tokens_per_sec"
UNIT = "tokens/s"
ENDE = dict(vocab=32000, emb=300, rnn=300, batch=256, tx=50, ty=50)
TRF = dict(vocab=32000, dim=512, ff=2048, depth=6, heads=8, batch=64, length=64)
CPU_SAMPLE_SENTENCES = 16
SEED = 2574600


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="ende", choices=["ende", "transformer"])
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-cuda-graph", action="store_true",
                    help="issue every kernel of a step from Python instead of replaying the captured step")
    ap.add_argument("--no-extras", action="store_true",
                    help="skip the secondary workloads (RNN decoding / transformer / beam-8 / captioning) at N=1")
    ap.add_argument("--extras", default="rnn_decode,transformer,beam,captioning,ende_realistic,ini_loop,late_gpu_checks")
    ap.add_argument("--no-dropout", action="store_true", help="transformer workload: keep_prob 1.0")
    ap.add_argument("--lengths", default="fixed", choices=["fixed", "realistic"],
                    help="en-de workload at N=1: 'realistic' draws sentence lengths from a clipped N(0.6 T, 0.2 T) "
                         "(SURVEY.md 8(d)); the tokens counted are the non-pad target tokens actually in the batches")
    ap.add_argument("--breakdown", action="store_true", help="print the per-entry-point time table")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (its losses and a fixed "
                         "sample of the updated parameters) to DIR/<name>.npy, to compare two builds output for output")
    return ap.parse_args()


def host_threads() -> int:
    """All the host cores the CPU arm may use.  torchrun exports OMP_NUM_THREADS=1 to its workers, which is
    not what a CPU baseline wants: the thread count is set explicitly, the same at every N."""
    n = os.cpu_count() or 1
    try:
        n = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        pass
    n = max(1, min(n, 64))
    torch.set_num_threads(n)
    return n


def workload_config(workload, n_gpus, batch, dropout=True):
    if workload == "transformer":
        return {"workload": "tests/transformer.ini at the perf shape: TransformerEncoder/Decoder L=6 d=512 h=8 "
                            "F=2048, tied embeddings, synthetic ids",
                "per_gpu_batch": batch, "global_batch": batch * n_gpus, "src_len": TRF["length"],
                "tgt_len": TRF["length"], "tokens_per_gpu_step": batch * TRF["length"], "vocab": TRF["vocab"],
                "optimizer": "LazyAdam beta2 0.98 eps 1e-9, Noam decay (lr 0.2, warmup 4000)",
                "dropout_keep_prob": 0.9 if dropout else 1.0, "lengths": "fixed (no padding)",
                "parallelism": "dp{}".format(n_gpus),
                "l2_between_iters": "parameters + optimizer state (4 x 245 MB) and activations exceed the 50 MB L2"}
    return {"workload": "examples/translation.ini GRU+Bahdanau en-de, synthetic ids",
            "per_gpu_batch": batch, "global_batch": batch * n_gpus, "src_len": ENDE["tx"], "tgt_len": ENDE["ty"],
            "vocab": ENDE["vocab"], "emb": 300, "rnn": 300, "optimizer": "Adam 1e-4, clip 1.0 per tensor, l2 1e-8",
            "lengths": "fixed (no padding)", "parallelism": "dp{}".format(n_gpus),
            "step_submission": "CrossEntropyTrainer(use_cuda_graph=True): the step is captured once per batch "
                               "shape and replayed; weight gradients are issued on a second stream inside the "
                               "captured backward pass (N>1: the bucketed NCCL all-reduce starts inside the "
                               "backward pass and is captured in the same graph)",
            "gemm": "wgmma: fp16 operands for the vocabulary projection and its gradients (fp32 accumulate), "
                    "tf32 elsewhere; GRU recurrences as persistent cluster kernels in exact fp32",
            "l2_between_iters": "working set per step (0.8 GB fp16 dlogits + 4 x 129 MB parameter buffers) "
                                "exceeds the 50 MB L2"}


def synthetic_batch(batch, seed, tx=ENDE["tx"], ty=ENDE["ty"], vocab=ENDE["vocab"], realistic=False):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(4, vocab, (batch, tx), generator=g)
    tgt = torch.randint(4, vocab, (batch, ty), generator=g)
    tgt[:, ty - 1] = 2  # </s>
    if realistic:
        # SURVEY.md 8(d), "realistic" variant: lengths ~ N(0.6 T, 0.2 T) clipped to [1, T]; the target length counts
        # its </s>; one full-length sentence per batch keeps the padded shape (pad_batch pads to the longest
        # sentence) - and with it the captured step - the same for every batch
        def lengths(limit):
            drawn = (torch.randn(batch, generator=g) * 0.2 * limit + 0.6 * limit).round().to(torch.int64)
            drawn = drawn.clamp(1, limit)
            drawn[0] = limit
            return drawn
        src_len, tgt_len = lengths(tx), lengths(ty)
        src[torch.arange(tx)[None, :] >= src_len[:, None]] = 0
        tgt.scatter_(1, (tgt_len - 1)[:, None], 2)
        tgt[torch.arange(ty)[None, :] >= tgt_len[:, None]] = 0
    return src, tgt


# ---------------------------------------------------------------------------
# CPU arm: the oracle restatement, timed
# ---------------------------------------------------------------------------
def cpu_ende_train(n_sent, steps, warmup, seed=SEED):
    """Full training steps of the oracle on n_sent sentences.  The op-for-op restatement is a mix of large
    products and very small tensor operations, for which more threads are not always faster: the first two
    untimed steps run with all cores and with half of them, the timed steps use the faster setting.
    Returns (tokens/s, seconds per step, threads used)."""
    from oracle import nm_oracle as O
    p = O.init_bahdanau_params(ENDE["vocab"], ENDE["vocab"], 300, 300, 300, 300, None, 300, False, seed=seed)
    spec = O.RNNDecoderSpec("decoder", "attention", ENDE["ty"], "tanh", False)
    st = O.AdamState(p)
    src, tgt = synthetic_batch(n_sent, seed)

    def one():
        t0 = time.perf_counter()
        O.train_step(p, spec, "sentence_encoder", src, tgt.t(), st, l2=1e-8, clip_norm=1.0)
        return time.perf_counter() - t0

    cores = host_threads()
    trial = {}
    for threads in sorted({cores, max(1, cores // 2)}, reverse=True):
        torch.set_num_threads(threads)
        trial[threads] = one()
    threads = min(trial, key=trial.get)
    torch.set_num_threads(threads)
    for _ in range(max(0, warmup - len(trial))):
        one()
    times = [one() for _ in range(steps)]
    per_step = sum(times) / len(times)
    # SURVEY.md 8(d)(a): the INIs all say num_threads=4 (tests/bahdanau.ini:23, examples/translation.ini:46) - one
    # more step at that setting, reported next to the headline CPU figure
    if threads == 4:
        FOUR_THREADS["tokens_per_sec"] = n_sent * ENDE["ty"] / per_step
    elif cores >= 4 and per_step * threads / 4 < 60.0:      # bounded: skipped where it would take minutes
        torch.set_num_threads(4)
        FOUR_THREADS["tokens_per_sec"] = n_sent * ENDE["ty"] / one()
        torch.set_num_threads(threads)
    else:
        FOUR_THREADS["tokens_per_sec"] = None
    return n_sent * ENDE["ty"] / per_step, per_step, threads


FOUR_THREADS = {}     # filled by cpu_ende_train: the same step with torch.set_num_threads(4)


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cores = host_threads()
    steps, warmup = max(1, min(args.steps, 3)), max(1, min(args.warmup, 2))
    if args.workload == "transformer":
        import bench_workloads
        batch = args.batch or TRF["batch"]
        n_sent = 4
        value, per_step = bench_workloads.cpu_transformer_train(n_sent, TRF["length"], steps, warmup)
        sample = "{} sentences x {} target tokens per step of the same model, {} timed steps".format(
            n_sent, TRF["length"], steps)
    else:
        batch = args.batch or ENDE["batch"]
        n_sent = batch                      # the whole per-GPU batch: about 5 s per step on the host cores
        value, per_step, cores = cpu_ende_train(n_sent, steps, warmup)
        sample = ("the full batch: {} sentences x {} target tokens per step, {} timed steps"
                  .format(n_sent, ENDE["ty"], steps))
    line = {"impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus,
            "steps": steps, "warmup": warmup, "ms_per_step": per_step * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args.workload, args.gpus, batch, not args.no_dropout),
            "cpu_sample_sentences_per_step": n_sent,
            "cpu_baseline": {"value": value, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
                             "note": "restated-reference CPU baseline (oracle/nm_oracle.py; TF 1.12 cannot be "
                                     "installed on this box); the thread count is set explicitly, the same at "
                                     "every N",
                             "value_with_4_threads": FOUR_THREADS.get("tokens_per_sec")},
            "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    emit(line)


# ---------------------------------------------------------------------------
# clocks sampler
# ---------------------------------------------------------------------------
class ClockSampler:
    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index = index
        self.samples = []
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._nvml = self._open_nvml(index)

    @staticmethod
    def _open_nvml(index):
        """An NVML handle of this process' GPU, opened ONCE before the timed region.  Polling through it costs
        microseconds; spawning `nvidia-smi` every 100 ms instead re-initialises NVML each time, which takes the
        driver's locks for tens of milliseconds and stalls this (and every other) process' launches - seen as 3-6 ms
        of host time per step in the device-resident loop.  None (-> the nvidia-smi fallback) if NVML is not usable."""
        try:
            import pynvml
            pynvml.nvmlInit()
            handle = None
            try:
                uuid = str(torch.cuda.get_device_properties(index).uuid)
                handle = pynvml.nvmlDeviceGetHandleByUUID(uuid if uuid.startswith("GPU-") else "GPU-" + uuid)
            except Exception:  # pylint: disable=broad-except
                visible = [v for v in os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",") if v.strip()]
                phys = int(visible[index]) if visible and all(v.strip().isdigit() for v in visible) else index
                handle = pynvml.nvmlDeviceGetHandleByIndex(phys)
            pynvml.nvmlDeviceGetClockInfo(handle, pynvml.NVML_CLOCK_SM)      # must answer, else fall back
            return pynvml, handle
        except Exception:  # pylint: disable=broad-except
            return None

    def _poll_nvml(self):
        pynvml, handle = self._nvml
        sm = pynvml.nvmlDeviceGetClockInfo(handle, pynvml.NVML_CLOCK_SM)
        sm_max = pynvml.nvmlDeviceGetMaxClockInfo(handle, pynvml.NVML_CLOCK_SM)
        try:
            power = pynvml.nvmlDeviceGetPowerUsage(handle) / 1000.0
        except Exception:  # pylint: disable=broad-except
            power = 0.0
        try:
            mask = pynvml.nvmlDeviceGetCurrentClocksEventReasons(handle)
        except Exception:  # pylint: disable=broad-except
            mask = pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(handle)

        def flag(bit):
            return "Active" if (mask & bit) else "Not Active"
        # hw_slowdown 0x8, hw_thermal_slowdown 0x40, sw_thermal_slowdown 0x20, sw_power_cap 0x4 (nvml.h)
        return [str(sm), str(sm_max), "{:.1f}".format(power), flag(0x8), flag(0x40), flag(0x20), flag(0x4)]

    def _run(self):
        while self._nvml is not None and not self._stop.is_set():
            try:
                self.samples.append(self._poll_nvml())
            except Exception:  # pylint: disable=broad-except
                self._nvml = None          # NVML stopped answering: fall through to nvidia-smi below
                break
            self._stop.wait(0.02)
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.FIELDS,
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True,
                                     timeout=5).stdout.strip()
                if out:
                    self.samples.append([x.strip() for x in out.split(",")])
            except Exception:  # pylint: disable=broad-except
                pass
            self._stop.wait(0.1)

    def __enter__(self):
        self._thread.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._thread.join(timeout=6)

    def summary(self):
        sm = sorted(int(float(s[0])) for s in self.samples if s and s[0].replace(".", "").isdigit())
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        reasons = set()
        for s in self.samples:
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                  "sw_power_cap"), s[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": int(float(self.samples[0][1])),
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:  # pylint: disable=broad-except
        return {}


DUMP_PARAM_SAMPLE = 4 << 20      # parameters written by --dump-outputs: 16 MB of float32


def dump_outputs(directory, out, arena):
    """The arrays a caller of the timed step receives - the step's losses (and regularisation sums) - and the
    parameters the step updated, as DIR/<name>.npy: float64 losses, float32 parameters (a fixed, seeded sample of
    the flat parameter buffer when it is larger than DUMP_PARAM_SAMPLE elements, in index order; the indices follow
    from SEED)."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    torch.cuda.synchronize()

    def values(x):
        items = x if isinstance(x, (list, tuple)) else [x]
        return np.concatenate([torch.as_tensor(v).detach().double().cpu().reshape(-1).numpy() for v in items])
    np.save(os.path.join(directory, "losses.npy"), values(out["losses"]))
    if out.get("l1l2") is not None:
        np.save(os.path.join(directory, "l1l2.npy"), values(out["l1l2"]))
    flat = arena.params.detach().reshape(-1)
    if flat.numel() > DUMP_PARAM_SAMPLE:
        g = torch.Generator().manual_seed(SEED)
        idx = torch.randperm(flat.numel(), generator=g)[:DUMP_PARAM_SAMPLE].sort().values
        flat = flat[idx.to(flat.device)]
    np.save(os.path.join(directory, "params_sample.npy"), flat.float().cpu().numpy())


def gemm_family_roofline(prof, prof_steps, xent_dims, peaks, total_ms):
    """The dominant kernel is tc_gemm_kernel (csrc/gemm_tc.cu): every dense projection, weight-gradient
    product and the fused vocabulary forward / backward are instances of it.  Algorithmic flops per launch =
    2*M*N*K of the product (DESIGN.md section 3); time = CUDA events around the launches inside the profiled
    steps.  Instances with fp16 operands are rated against the fp16/bf16 peak, tf32 instances
    cannot exceed half of it (the ceiling is reported too)."""
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))
    peak_src = "measured bf16_tflops_sustained (MEASURED_PEAKS.json)" if peaks else \
        "H100 SXM data sheet, dense fp16/bf16 at 700 W"
    m, k, v = xent_dims
    fam_flops = fam_ms = f16_flops = f16_ms = 0.0
    instances = []
    for name, d in prof.items():
        fl = None
        mm = re.match(r"nm_gemm\[(\w\w) (\d+)x(\d+)x(\d+)\]", name)
        if mm:
            fl = 2.0 * int(mm.group(2)) * int(mm.group(3)) * int(mm.group(4))
        elif name.split("[")[0] in ("nm_logits_xent_fwd", "nm_logits_xent_bwd", "nm_logits_xent_fwd16",
                                    "nm_logits_xent_bwd16"):
            fl = 2.0 * m * k * v
        else:
            mm = re.match(r"nm_gemm_f16(?:_tn)?\[(\d+)x(\d+)x(\d+)\]", name)
            if mm:
                fl = 2.0 * int(mm.group(1)) * int(mm.group(2)) * int(mm.group(3))
        if fl is None:
            continue
        calls = d["calls"]
        kind = "f16" if "16" in name.split("[")[0] else "tf32"
        fam_flops += fl * calls
        fam_ms += d["ms"]
        if kind == "f16":
            f16_flops += fl * calls
            f16_ms += d["ms"]
        instances.append({"call": name, "launches_per_step": calls // prof_steps,
                          "ms_per_launch": d["ms"] / calls, "tflops": fl / (d["ms"] / calls * 1e-3) / 1e12,
                          "kind": kind})
    if fam_ms <= 0:
        return None
    instances.sort(key=lambda e: -e["ms_per_launch"] * e["launches_per_step"])
    ach = fam_flops / (fam_ms * 1e-3) / 1e12
    roof = {"kernel": "tc_gemm_kernel (wgmma; all instances of the step: fp16 vocabulary products, "
                      "tf32 elsewhere)",
            "bound": "tensor", "achieved": ach, "peak": peak_tf, "unit": "TFLOP/s", "frac": ach / peak_tf,
            "peak_source": peak_src,
            "share_of_step": fam_ms / prof_steps / max(total_ms, 1e-9),
            "instances": instances[:8]}
    if f16_ms > 0:
        roof["f16_instances"] = {"achieved": f16_flops / (f16_ms * 1e-3) / 1e12,
                                 "frac": f16_flops / (f16_ms * 1e-3) / 1e12 / peak_tf,
                                 "share_of_family_time": f16_ms / fam_ms}
    return roof


# ---------------------------------------------------------------------------
# GPU arm
# ---------------------------------------------------------------------------
def run_b200(args):
    import bench_models
    from neuralmonkey_b200 import distributed, lib
    distributed.init_from_env()
    rank, world = distributed.rank(), distributed.world_size()
    workload = args.workload
    graph = not args.no_cuda_graph
    if workload == "transformer":
        batch = args.batch or TRF["batch"]
        model = bench_models.build_transformer(vocab=TRF["vocab"], max_len=TRF["length"], cuda_graph=graph,
                                               dropout=not args.no_dropout)
        feed = bench_models.feed_transformer
        tx = ty = TRF["length"]
        xent_dims = (batch * ty, TRF["dim"], TRF["vocab"])
    else:
        batch = args.batch or ENDE["batch"]
        model = bench_models.build_ende(vocab=ENDE["vocab"], cuda_graph=graph)
        feed = bench_models.feed_ende
        tx, ty = ENDE["tx"], ENDE["ty"]
        xent_dims = (batch * ty, 300, ENDE["vocab"])
    trainer = model.trainer
    dev = model.arena.params.device
    tokens_per_step_rank = batch * ty
    realistic = args.lengths == "realistic"
    if realistic and (world > 1 or workload != "ende"):
        raise SystemExit("--lengths realistic is an N=1 variant of the en-de workload")

    # a few distinct synthetic batches, resident on the device (value) and pinned on host (e2e)
    host_batches = [synthetic_batch(batch, SEED + rank + 1000 * i, tx, ty, realistic=realistic) for i in range(4)]
    pinned = [(s.pin_memory(), t.pin_memory()) for s, t in host_batches]
    # decoder ids stay on the host: feed_ids derives the teacher-forcing inputs there (a few microseconds of
    # integer work) and uploads both id tensors through pinned staging
    dev_batches = [(s.to(dev), t) for s, t in host_batches]

    def step_device_inputs(i):
        src, tgt = dev_batches[i % len(dev_batches)]
        feed(model, src, tgt, True)
        return trainer.train_step()

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    host_ms = [0.0]
    last_out = [None]

    def timed(step_fn, steps, read_loss):
        barrier()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        last = None
        t_host = time.perf_counter()
        for i in range(steps):
            out = step_fn(i)
            last_out[0] = out
            if read_loss:
                last = float(out["losses"][0])  # device -> host read of the step's loss
        host_ms[0] = (time.perf_counter() - t_host) * 1e3 / steps   # time the host needs to ENQUEUE a step
        ev1.record()
        barrier()
        ms = torch.tensor([ev0.elapsed_time(ev1)], device=dev)
        if world > 1:
            torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
        return float(ms) / steps, last

    for i in range(max(args.warmup, 3)):
        step_device_inputs(i)
    # rank 0 alone samples the clocks (its line is the one printed): eight ranks polling nvidia-smi at once
    # contend for the driver and stall each other's launches (seen as 6 ms of host time per step at N=8)
    with (ClockSampler(dev.index or 0) if rank == 0 else contextlib.nullcontext()) as clocks:
        ms_step, _ = timed(step_device_inputs, args.steps, read_loss=False)
    host_enqueue_ms = host_ms[0]
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last_out[0], model.arena)

    # per-entry-point device time (CUDA events around every C-ABI call) and the kernel count of a step: these
    # steps issue every launch from Python - a replayed graph contains the same kernel nodes but does not
    # pass through the library's launch counter
    graphed = trainer.use_cuda_graph
    trainer.use_cuda_graph = False
    launches0 = lib.launch_count()
    lib.profile_start()
    prof_steps = min(args.steps, 5)
    for i in range(prof_steps):
        step_device_inputs(i)
    prof = lib.profile_stop()
    launches = (lib.launch_count() - launches0) // prof_steps * args.steps
    trainer.use_cuda_graph = graphed

    def step_e2e(i):
        src, tgt = pinned[i % len(pinned)]
        feed(model, src, tgt, True)   # H2D of the pinned id tensors inside the timed region
        return trainer.train_step()

    for i in range(3):
        step_e2e(i)
    ms_e2e, loss = timed(step_e2e, args.steps, read_loss=True)
    exposed_comm_ms = getattr(trainer, "min_exposed_comm_ms", None)

    if rank != 0:
        return
    value = world * tokens_per_step_rank / (ms_step * 1e-3)
    e2e_value = world * tokens_per_step_rank / (ms_e2e * 1e-3)
    if realistic:
        # the tokens that were in the timed batches: non-pad target positions (sum of train_mask, </s> included)
        tgt_tokens = [int((t != 0).sum()) for _s, t in host_batches]
        src_tokens = [int((s_ != 0).sum()) for s_, _t in host_batches]
        timed = [i % len(host_batches) for i in range(args.steps)]
        mean_tgt = sum(tgt_tokens[i] for i in timed) / len(timed)
        mean_src = sum(src_tokens[i] for i in timed) / len(timed)
        value, e2e_value = mean_tgt / (ms_step * 1e-3), mean_tgt / (ms_e2e * 1e-3)
        line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": 1, "steps": args.steps,
                "warmup": max(args.warmup, 3), "ms_per_step": ms_step, "higher_is_better": True,
                "lengths": "realistic: N(0.6 T, 0.2 T) clipped to [1, T], one full-length sentence per batch",
                "target_tokens_per_step": mean_tgt, "source_tokens_per_step": mean_src,
                "padded_positions_per_step": batch * ty,
                "source_plus_target_tokens_per_sec": (mean_src + mean_tgt) / (ms_step * 1e-3),
                "e2e": {"value": e2e_value, "unit": UNIT, "ms_per_step": ms_e2e,
                        "h2d_bytes_per_step": 2 * batch * (tx + ty) * 8, "d2h_bytes_per_step": 4, "last_loss": loss},
                "clocks": clocks.summary(), "config": workload_config(workload, world, batch)}
        line["config"]["lengths"] = line["lengths"]
        emit(line)
        bench_models.cleanup()
        return

    peaks = measured_peaks()
    table = sorted(((n, d["ms"] / prof_steps, d["calls"] // prof_steps) for n, d in prof.items()),
                   key=lambda x: -x[1])
    total_ms = sum(t for _, t, _ in table)
    roof = gemm_family_roofline(prof, prof_steps, xent_dims, peaks, total_ms)
    if args.breakdown:
        for n, t, c in table:
            print("# {:40s} {:8.3f} ms/step  {:4d} calls/step".format(n, t, c), file=sys.stderr)
        print("# sum {:.3f} ms of device time vs {:.3f} ms per step".format(total_ms, ms_step), file=sys.stderr)

    cpu = parity = None
    if not args.no_cpu_baseline and world == 1:
        cores = host_threads()
        if workload == "ende":
            cpu_value, cpu_step, cores = cpu_ende_train(batch, 1, 2)
            cpu = {"value": cpu_value, "unit": UNIT, "cores": cores, "kind": "port",
                   "sample": "the full batch: {} sentences x {} target tokens per step, 1 timed step ({:.1f} s) "
                             "after 2 untimed ones".format(batch, ty, cpu_step),
                   "value_with_4_threads": FOUR_THREADS.get("tokens_per_sec")}
            parity = ende_parity(model, feed)
        else:
            import bench_workloads
            cpu_value, cpu_step = bench_workloads.cpu_transformer_train(4, ty, 2, 1)
            cpu = {"value": cpu_value, "unit": UNIT, "cores": cores, "kind": "port",
                   "sample": "4 sentences x {} target tokens per step, 2 timed steps ({:.1f} s each)"
                             .format(ty, cpu_step)}

    # the other configurations of BASELINE.json; N=1 only, a few seconds each
    extras = None
    if world == 1 and not args.no_extras and workload == "ende":
        import bench_workloads
        extras = {}
        del model
        torch.cuda.empty_cache()
        for name in [n for n in args.extras.split(",") if n]:
            t_extra = time.perf_counter()
            try:
                extras[name] = bench_workloads.RUNNERS[name](cpu=not args.no_cpu_baseline)
            except Exception as exc:  # pylint: disable=broad-except
                import traceback
                traceback.print_exc()
                extras[name] = {"error": "{}: {}".format(type(exc).__name__, exc)}
            if isinstance(extras[name], dict):
                extras[name]["wall_s"] = round(time.perf_counter() - t_extra, 1)
            torch.cuda.empty_cache()

    h2d = 2 * batch * (tx + ty) * 8  # int64 ids: encoder ids, decoder targets + fed symbols
    line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": max(args.warmup, 3), "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None,
            "dtype": "f32 storage; tensor-core products in fp16 (vocabulary) / tf32 with fp32 accumulation",
            "data": "synthetic", "config": workload_config(workload, world, batch, not args.no_dropout),
            "e2e": {"value": e2e_value, "unit": UNIT, "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "last_loss": loss},
            "gpu_launches": launches,
            "gpu_launches_note": "kernels of libnmb200 per step x timed steps, counted by nm_launch_count() over "
                                 "eagerly issued steps" + (" (the timed steps replay the same kernels as one "
                                                           "captured CUDA graph per step)" if graphed else ""),
            "clocks": clocks.summary(), "roofline": roof, "cpu_baseline": cpu, "parity": parity,
            "breakdown_ms_per_step": {n: round(t, 4) for n, t, _ in table[:18]},
            "host_enqueue_ms_per_step": host_enqueue_ms,
            "exposed_comm_ms_per_step": exposed_comm_ms,
            "exposed_comm_note": "device time the compute stream waits for the gradient exchange after the backward "
                                 "pass, minimum over the eagerly issued profile steps (eager steps drift apart by "
                                 "host jitter, so this includes waiting for the slowest rank; the graph-replayed "
                                 "steps the headline times do not drift)" if world > 1 else None,
            "extra_workloads": extras}
    emit(line)
    bench_models.cleanup()


def ende_parity(model, feed):
    """The benched engine (wgmma fp16/tf32 products, cluster GRU, CUDA-graph step) against the fp32
    oracle at the perf dims (H = E = 300, V = 32000, T = 50) on the CPU arm's 16-sentence sample, with O(0.1)
    random parameters so that every activation matters: train loss within 1e-3 (north_star)."""
    from oracle import nm_oracle as O
    arena = model.arena
    shapes = {n: torch.zeros(arena.variables[n].shape) for n in sorted(arena.order)}
    params = O.randomize(shapes, scale=0.1, seed=11)
    for name in params:
        if name.endswith("gamma"):
            params[name] = 1.0 + params[name]
    arena.load_dict(params)
    src, tgt = synthetic_batch(CPU_SAMPLE_SENTENCES, SEED + 77)
    feed(model, src.pin_memory(), tgt.pin_memory(), True)
    gpu_loss = float(model.decoder.train_loss)
    spec = O.RNNDecoderSpec("decoder", "attention_sentence_encoder", ENDE["ty"], "tanh", False)
    with torch.no_grad():
        oenc = O.sentence_encoder(params, "sentence_encoder", src)
        odec = O.decoder_train(params, spec, oenc, tgt.t())
    want = float(odec["train_loss"])
    return {"what": "train loss of the benched engine vs the fp32 CPU oracle, en-de dims, 16 sentences x 50",
            "gpu_loss": gpu_loss, "oracle_loss": want, "abs_diff": abs(gpu_loss - want), "tolerance": 1e-3,
            "ok": abs(gpu_loss - want) < 1e-3}


_REAL_STDOUT = None


def emit(line):
    """The ONE JSON line, written to the process's original stdout."""
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        os.write(_REAL_STDOUT, data)


def main():
    # Libraries (NCCL prints its version banner) write to file descriptor 1: keep the real stdout
    # for the JSON line only and send everything else to stderr.
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    args = parse_args()
    if args.impl == "reference":
        run_reference(args)
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: neuralmonkey_b200 has no CPU path "
                         "(use --impl reference for the CPU restatement)")
    run_b200(args)


if __name__ == "__main__":
    main()
