"""Time the four cluster-GRU calls of an en-de training step (encoder fwd/bwd pair, decoder fwd/bwd) at
B=256, T=50, H=300 with CUDA events, print the per-phase cycle counters of thread 0 of CTA 0
(nm_gru_debug_profile), and check that every build given computes what the first one does within the exact
tolerances of the cluster GRU tests (max-abs 2e-5 on the forward outputs, relative 5e-5 on the gradients): builds
that group the reduction differently differ in the last bits.

    python tools/gru_plan_bench.py [--lib A.so --lib B.so ...] [--rounds 5] [--reps 20]

Each --lib is a build of libnmb200.so (default: the one in the tree); the rounds alternate between them, so
two builds are compared in one session on the same card.  The card's name, power limit and SM clock are
read in the same run."""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralmonkey_b200 import lib as nmlib  # noqa: E402

B, T, H = 256, 50, 300
FWD_SLOTS = ("wait_h", "sync+prefetch", "phase1", "wait_rh", "phase2")
BWD_SLOTS = ("wait_dzc_dzu", "sync+prefetch", "G1", "wait_dzr", "sync", "G2+E1")


def load(path):
    handle = ctypes.CDLL(path)
    restypes = {"s": ctypes.c_char_p, "l": ctypes.c_int64, "i": ctypes.c_int}
    for name, (rcode, codes) in nmlib.parse_header().items():
        fn = getattr(handle, name)
        fn.restype = restypes[rcode]
        fn.argtypes = [nmlib._CTYPES[c] for c in codes]
    return handle


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip() or torch.cuda.get_device_name(0)


def inputs():
    g = torch.Generator().manual_seed(0)
    d = {}

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).cuda()
    for s in ("a", "b", "d"):  # encoder directions a, b and the decoder
        d["x" + s] = rnd(B, T, 3 * H, scale=0.5)
        d["wg" + s] = rnd(H, 2 * H, scale=H ** -0.5)
        d["wc" + s] = rnd(H, H, scale=H ** -0.5)
        d["ds" + s] = rnd(B, T, H)
        d["df" + s] = rnd(B, H)
        for n, k in (("states", 1), ("gates", 3), ("hprev", 1), ("rh", 1), ("dx", 3)):
            d[n + s] = torch.empty(B, T, k * H, device="cuda")
        d["final" + s] = torch.empty(B, H, device="cuda")
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0] = T
    d["len"] = lengths.cuda()
    d["h0"] = rnd(B, H, scale=0.5)
    d["mask"] = ((torch.rand(B, T, H, generator=g) < 0.7).float() / 0.7).cuda()
    d["raw"] = torch.empty(B, T, H, device="cuda")
    d["dh0"] = torch.empty(B, H, device="cuda")
    d["work"] = torch.empty(2 * B * H, device="cuda")
    return d


def calls(h, d):
    p = nmlib.ptr
    st = 0  # the legacy default stream, shared by every build loaded in the process

    def check(rc):
        if rc:
            raise RuntimeError(h.nm_last_error().decode())

    def enc_fwd():
        check(h.nm_gru_seq_fwd_pair(
            p(d["xa"]), p(d["wga"]), p(d["wca"]), 0, p(d["statesa"]), p(d["finala"]), p(d["gatesa"]),
            p(d["hpreva"]), p(d["rha"]),
            p(d["xb"]), p(d["wgb"]), p(d["wcb"]), 1, p(d["statesb"]), p(d["finalb"]), p(d["gatesb"]),
            p(d["hprevb"]), p(d["rhb"]), p(d["len"]), B, T, H, st))

    def enc_bwd():
        check(h.nm_gru_seq_bwd_pair(
            p(d["wga"]), p(d["wca"]), 0, p(d["gatesa"]), p(d["hpreva"]), p(d["dsa"]), p(d["dfa"]), p(d["dxa"]),
            p(d["wgb"]), p(d["wcb"]), 1, p(d["gatesb"]), p(d["hprevb"]), p(d["dsb"]), p(d["dfb"]), p(d["dxb"]),
            p(d["len"]), p(d["work"]), B, T, H, st))

    def dec_fwd():
        check(h.nm_gru_seq_fwd(p(d["xd"]), p(d["wgd"]), p(d["wcd"]), p(d["h0"]), None, p(d["mask"]), 0,
                               p(d["statesd"]), p(d["raw"]), p(d["finald"]), p(d["gatesd"]), p(d["hprevd"]),
                               p(d["rhd"]), B, T, H, 0, st))

    def dec_bwd():
        check(h.nm_gru_seq_bwd(p(d["wgd"]), p(d["wcd"]), None, p(d["mask"]), 0, p(d["gatesd"]), p(d["hprevd"]),
                               p(d["dsd"]), None, p(d["dfd"]), p(d["dxd"]), p(d["dh0"]), p(d["work"]), B, T, H,
                               0, st))
    return {"enc_fwd_pair": enc_fwd, "enc_bwd_pair": enc_bwd, "dec_fwd": dec_fwd, "dec_bwd": dec_bwd}


OUTPUTS = ("statesa", "finala", "statesb", "finalb", "statesd", "raw", "finald", "gatesd", "dxa", "dxb", "dxd", "dh0")
GRADIENTS = ("dxa", "dxb", "dxd", "dh0")
TOL, GTOL = 2e-5, 5e-5  # tests/test_gpu_gru_cluster.py


def compare(ref, got):
    """{output: (max-abs difference, relative difference, within tolerance)}"""
    out = {}
    for o in OUTPUTS:
        a, b = got[o].double(), ref[o].double()
        mad = float((a - b).abs().max())
        rel = float((a - b).norm() / (b.norm() + 1e-30))
        out[o] = (mad, rel, rel < GTOL if o in GRADIENTS else mad < TOL)
    return out


def run_all(fns):
    for f in fns.values():
        f()


def timed(fns, reps):
    ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in fns}
    for n, f in fns.items():
        ev[n][0].record()
        for _ in range(reps):
            f()
        ev[n][1].record()
    torch.cuda.synchronize()
    return {n: e0.elapsed_time(e1) / reps for n, (e0, e1) in ev.items()}


def phases(h, fns, prof, reps=4):
    out = {}
    for n, f in fns.items():
        slots = FWD_SLOTS if "fwd" in n else BWD_SLOTS
        calls_per = 2 if "pair" in n else 1
        prof.zero_()
        h.nm_gru_debug_profile(prof.data_ptr())
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
        h.nm_gru_debug_profile(None)
        c = prof.cpu().tolist()
        div = reps * calls_per * T
        out[n] = " ".join("%s=%d" % (s, v / div) for s, v in zip(slots, c)) + "  total=%d" % (sum(c) / div)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="libnmb200.so build to time (repeatable)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20, help="launches of each call per timed window")
    args = ap.parse_args()
    paths = args.lib or [nmlib.LIB_PATH]
    torch.cuda.init()
    libs = [load(p) for p in paths]
    print("card (name, power limit, SM clock, max SM clock):", card())
    d = inputs()
    ref = None
    for path, h in zip(paths, libs):
        print("%s: resident clusters fwd/bwd %d/%d" % (path, h.nm_gru_resident_clusters(0),
                                                      h.nm_gru_resident_clusters(1)))
        for o in OUTPUTS:
            d[o].fill_(float("nan"))
        run_all(calls(h, d))
        torch.cuda.synchronize()
        got = {o: d[o].clone() for o in OUTPUTS}
        if ref is None:
            ref = got
        else:
            diff = compare(ref, got)
            same = all(torch.equal(ref[o], got[o]) for o in OUTPUTS)
            print("  against %s: bit-identical %s, within the exact tolerances %s" % (
                paths[0], same, all(ok for _, _, ok in diff.values())))
            print("    " + "  ".join("%s %.1e/%.1e%s" % (o, m, r, "" if ok else " (OVER)")
                                     for o, (m, r, ok) in diff.items()) + "   (max-abs/relative)")
    fns = [calls(h, d) for h in libs]
    for f in fns:  # warm-up
        timed(f, 2)
    times = [[] for _ in libs]
    for r in range(args.rounds):
        for i, f in enumerate(fns):
            t = timed(f, args.reps)
            times[i].append(t)
            print("round %d  %-40s " % (r, os.path.relpath(paths[i])) +
                  "  ".join("%s %.3f" % (n, v) for n, v in t.items()) + "  | four calls %.3f ms" % sum(t.values()),
                  flush=True)
    for i, p in enumerate(paths):
        tot = sorted(sum(t.values()) for t in times[i])
        print("%s: four calls %.3f-%.3f ms (median %.3f) over %d rounds" % (p, tot[0], tot[-1], tot[len(tot) // 2],
                                                                             len(tot)))
    prof = torch.zeros(8, dtype=torch.int64, device="cuda")
    for p, h, f in zip(paths, libs, fns):
        print("cycles/step of thread 0 of CTA 0, %s:" % p)
        for n, s in phases(h, f, prof).items():
            print("   %-13s %s" % (n, s))
    print("card after the run:", card())


if __name__ == "__main__":
    main()
