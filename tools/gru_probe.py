"""Time the cluster GRU recurrence forward and backward (nm_gru_seq_fwd / nm_gru_seq_bwd) at the en-de shape
and print the per-phase cycle counters of thread 0 of CTA 0 (nm_gru_debug_profile), per step."""
import os, sys, torch
sys.path.insert(0, ".")
from neuralmonkey_b200 import lib
from neuralmonkey_b200.lib import call, ptr
torch.manual_seed(0)
H, T = 300, 50
FWD_SLOTS = ("wait_h", "sync+prefetch", "phase1", "wait_rh", "phase2")
BWD_SLOTS = ("wait_dzc_dzu", "sync+prefetch", "G1", "wait_dzr", "sync", "G2+E1")


def run(B, budget, reps=3):
    dev = "cuda"
    xproj = torch.randn(B, T, 3 * H, device=dev) * 0.1
    wg = torch.randn(H, 2 * H, device=dev) * 0.05
    wc = torch.randn(H, H, device=dev) * 0.05
    states = torch.empty(B, T, H, device=dev); final = torch.empty(B, H, device=dev)
    gates = torch.empty(B, T, 3 * H, device=dev); hprev = torch.empty(B, T, H, device=dev)
    rh = torch.empty(B, T, H, device=dev)
    dstates = torch.randn(B, T, H, device=dev); dfinal = torch.randn(B, H, device=dev)
    dxproj = torch.empty(B, T, 3 * H, device=dev); work = torch.empty(2 * B * H, device=dev)

    def fwd():
        call("nm_gru_seq_fwd", ptr(xproj), ptr(wg), ptr(wc), None, None, None, 0, ptr(states), None, ptr(final),
             ptr(gates), ptr(hprev), ptr(rh), B, T, H, budget, lib.stream())

    def bwd():
        call("nm_gru_seq_bwd", ptr(wg), ptr(wc), None, None, 0, ptr(gates), ptr(hprev), ptr(dstates), None,
             ptr(dfinal), ptr(dxproj), None, ptr(work), B, T, H, budget, lib.stream())

    out = {}
    for name, go in (("fwd", fwd), ("bwd", bwd)):
        go(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): go()
        e1.record(); torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
    return out, fwd, bwd


def phases(go, names, prof, reps=4):
    prof.zero_()
    lib.load().nm_gru_debug_profile(prof.data_ptr())
    for _ in range(reps): go()
    torch.cuda.synchronize()
    lib.load().nm_gru_debug_profile(None)
    c = prof.cpu().tolist()
    tot = sum(c)
    return " ".join("%s=%d" % (n, v / (reps * T)) for n, v in zip(names, c)) + "  total=%d" % (tot / (reps * T))


print("device:", torch.cuda.get_device_name(0))
print("resident clusters fwd/bwd:", lib.load().nm_gru_resident_clusters(0), lib.load().nm_gru_resident_clusters(1))
prof = torch.zeros(8, dtype=torch.int64, device="cuda")
for B, budget in ((16, 8), (256, 132)):
    ms, fwd, bwd = run(B, budget)
    for name, go, names in (("fwd", fwd, FWD_SLOTS), ("bwd", bwd, BWD_SLOTS)):
        print("B=%4d budget=%3d %s -> %.3f ms  (%.1f us/step)" % (B, budget, name, ms[name], ms[name] * 1000 / T),
              flush=True)
        print("   cycles/step: " + phases(go, names, prof), flush=True)
