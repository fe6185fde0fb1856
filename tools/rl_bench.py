"""Timings of the reinforcement-learning objectives on the GPU (one JSON line).

* `nm_sentence_ngram_reward` at B = 256 and 512, T = 50, against the host restatement of the reference's
  sentence_bleu (tests/rl_oracle.py, tuple-keyed Counters);
* `nm_sample_logits_step` at 256 x 32000 against the time of reading the logits once at 3.35 TB/s;
* eager training steps of the en-de bench model (B = 256, T = 50, V = 32000): cross-entropy, cross-entropy +
  self-critical (weights 0.5 / 0.5, as tests/self-critical.ini) and REINFORCE with sample_size = 2 (GLEU rewards,
  baseline, ce_smoothing = 0.5, as tests/rl.ini), each with a breakdown of one step: the forward pass with the
  decoding loops, the backward pass, the rewards and the sampling.  The </s> bias is pushed down so that every
  loop runs its 50 steps, the length of the cross-entropy pass.

    python tools/rl_bench.py [--steps 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def bench_rewards(out):
    from neuralmonkey_b200 import ops
    from tests import rl_oracle
    rng = np.random.RandomState(0)
    for bsz in (256, 512):
        refs = rng.randint(4, 2000, size=(50, bsz)).astype(np.int64)
        hyps = np.where(rng.rand(50, bsz) < 0.5, refs, rng.randint(4, 2000, size=(50, bsz))).astype(np.int64)
        r, h = torch.from_numpy(refs).cuda(), torch.from_numpy(hyps).cuda()
        ms = _events(lambda: ops.sentence_ngram_reward(r, h, "bleu"), 200)
        t0 = time.perf_counter()
        rl_oracle.sentence_bleu(refs, hyps)
        host_ms = (time.perf_counter() - t0) * 1e3
        out["reward_B{}_T50".format(bsz)] = {"kernel_ms": ms, "host_restatement_ms": host_ms}


def bench_sampler(out):
    from neuralmonkey_b200 import ops
    logits = torch.randn(256, 32000, device="cuda")
    fin = torch.zeros(256, dtype=torch.bool, device="cuda")
    ms = _events(lambda: ops.sample_logits_step(logits, 1.0, fin, 3, 0, 0), 200)
    bound = logits.numel() * 4 / HBM_BYTES_PER_S * 1e3
    out["sampler_256x32000"] = {"kernel_ms": ms, "read_once_bound_ms": bound, "share_of_bound": bound / ms}


def bench_steps(out, steps):
    import bench_models as bm
    from neuralmonkey_b200 import lib, runtime
    from neuralmonkey_b200.evaluators.gleu import GLEUEvaluator
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from neuralmonkey_b200.trainers.objective import CostObjective
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    model = bm.build_ende(cuda_graph=False)
    dec = model.decoder
    with torch.no_grad():
        dec.decoding_b[2] = -1e3
    src, tgt = bm.synthetic_ids(256, 50, 32000, seed=1), bm.synthetic_ids(256, 50, 32000, seed=2)
    rl = ReinforceObjective(dec, GLEUEvaluator(), subtract_baseline=True, sample_size=2, ce_smoothing=0.5)
    host_reward_s = []
    score = rl.score_with_reward_function

    def timed_score(refs, hyps):
        t0 = time.perf_counter()
        res = score(refs, hyps)
        host_reward_s.append(time.perf_counter() - t0)
        return res
    rl.score_with_reward_function = timed_score
    configs = {"ce": [CostObjective(dec)],
               "self_critical": [CostObjective(dec, 0.5), SelfCriticalObjective(dec, sentence_bleu, weight=0.5)],
               "reinforce_s2": [rl]}
    for name, objectives in configs.items():
        trainer = GenericTrainer(objectives, l2_weight=1e-8, clip_norm=1.0)

        def step():
            bm.feed_ende(model, src, tgt, train=True)
            return trainer.train_step()
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            losses = step()["losses"]
        torch.cuda.synchronize()
        entry = {"step_ms": (time.perf_counter() - t0) * 1e3 / steps, "losses": [float(v) for v in losses]}
        # one more step, phase by phase, with the device time of every entry point
        bm.feed_ende(model, src, tgt, train=True)
        del host_reward_s[:]
        lib.profile_start()
        runtime.advance_dropout()
        runtime.arena().zero_grad()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        total = None
        for obj in objectives:
            term = obj.loss * (1.0 if obj.weight is None else obj.weight)
            total = term if total is None else total + term
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        total.backward()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        prof = lib.profile_stop()
        rewards_dev = prof.get("nm_sentence_ngram_reward", {}).get("ms", 0.0)
        sampling_dev = prof.get("nm_sample_logits_step", {}).get("ms", 0.0)
        entry.update({
            "forward_with_loops_ms": (t1 - t0) * 1e3, "backward_ms": (t2 - t1) * 1e3,
            "rewards_device_ms": rewards_dev, "rewards_host_ms": sum(host_reward_s) * 1e3,
            "sampling_device_ms": sampling_dev,
            "rl_kernels_share_of_step": (rewards_dev + sampling_dev) / entry["step_ms"],
            "nm_gru_seq_fwd_calls": prof.get("nm_gru_seq_fwd", {}).get("calls", 0)})
        out["step_" + name] = entry
    bm.cleanup()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rl_bench needs a CUDA device")
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit"] = "unknown"
    bench_rewards(out)
    bench_sampler(out)
    bench_steps(out, args.steps)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as handle:
            handle.write(line + "\n")


if __name__ == "__main__":
    main()
