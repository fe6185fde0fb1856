import os, sys, time, torch
sys.path.insert(0, ".")
from neuralmonkey_b200 import lib, ops
from neuralmonkey_b200.lib import call, ptr
torch.manual_seed(0)
H, T = 300, 50
def run(B, budget, reps=3):
    dev = "cuda"
    xproj = torch.randn(B, T, 3 * H, device=dev) * 0.1
    wg = torch.randn(H, 2 * H, device=dev) * 0.05
    wc = torch.randn(H, H, device=dev) * 0.05
    states = torch.empty(B, T, H, device=dev); final = torch.empty(B, H, device=dev)
    gates = torch.empty(B, T, 3 * H, device=dev); hprev = torch.empty(B, T, H, device=dev); rh = torch.empty(B, T, H, device=dev)
    def go():
        call("nm_gru_seq_fwd", ptr(xproj), ptr(wg), ptr(wc), None, None, None, 0, ptr(states), None, ptr(final),
             ptr(gates), ptr(hprev), ptr(rh), B, T, H, budget, lib.stream())
    go(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): go()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
print("resident clusters fwd/bwd:", lib.load().nm_gru_resident_clusters(0), lib.load().nm_gru_resident_clusters(1))
prof = torch.zeros(8, dtype=torch.int64, device="cuda")
lib.load().nm_gru_debug_profile(prof.data_ptr())
for B, budget in ((16, 8), (256, 132)):
    ms = run(B, budget)
    print("B=%4d budget=%3d -> %.3f ms  (%.1f us/step)" % (B, budget, ms, ms * 1000 / T), flush=True)
    c = prof.cpu().tolist(); prof.zero_()
    tot = sum(c)
    print("   cycles/step: " + " ".join("%s=%d" % (n, v / (4 * T)) for n, v in zip(("load1","dot1","ew1","bar1","load2","dot2","ew2","bar2"), c)), "total=%d" % (tot / (4 * T)))
os.environ["NMB200_GRU"] = "steps"
