"""Check the learner's fc1 products against fp64 on the same operands, and time them: the forward
(iplan_learner_fc1_forward: feature LayerNorm folded into fc1 of actor and critic) and the backward
(iplan_learner_fc1_backward: G = dZ1^T X and the fc1.weight / feature_norm gradients).

    python tools/check_fc1.py            # a ragged small case, one agent at full width, the bench shape

At the bench shape it also times the two product kernels alone (torch.profiler, several launches) and prints the rate of
the X stream (Xh + Xl, 4 bytes per element, read once per product) against the H100 SXM's 3.35 TB/s of HBM3, and the
rate of the tensor work (three f16 products per fp32 product).
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iplan_b200 import _lib                          # noqa: E402
from iplan_b200.modules.flat import ParamStack       # noqa: E402


HBM_TBS = 3.35                                       # H100 SXM data sheet


def kernel_ms(call, name, reps):
    """Mean device time of the kernels whose name contains `name`, over `reps` calls."""
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
             for e in prof.key_averages() if name in e.key)
    return us / 1e3 / reps


def rates(what, ms, A, rows, Fp):
    x_bytes = A * rows * Fp * 4                      # Xh + Xl
    flops = 3 * 2 * A * rows * 128 * Fp              # hi*hi + lo*hi + hi*lo
    gbs = x_bytes / ms / 1e6
    print(f"  {what} kernel: {ms:.3f} ms; X stream {gbs:.0f} GB/s = {gbs / (HBM_TBS * 1e3):.0%} of {HBM_TBS} TB/s; "
          f"tensor work {flops / ms / 1e9:.0f} TFLOP/s", flush=True)


def run(A, rows, F, n_act=5, reps=5, kernel_rates=False):
    """Largest error relative to the fp64 result's magnitude, over the forward Z1 and the backward G."""
    torch.manual_seed(0)
    dev = "cuda"
    Fp = (F + 31) // 32 * 32
    actor = ParamStack("actor", A, (F, n_act), device=dev)
    critic = ParamStack("critic", A, (F,), device=dev)
    for st in (actor, critic):
        st.flat.copy_(torch.randn_like(st.flat) * 0.1)
    X = torch.zeros(A, rows, Fp, device=dev)
    X[..., :F] = torch.rand(A, rows, F, device=dev) * 2 - 1
    P, lib, st = _lib.ptr, _lib.lib, _lib.stream()
    z = lambda *s, **k: torch.zeros(*s, device=dev, **k)
    hz = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float16)
    stat, Xh, Xl = z(A, rows, 2), hz(A, rows, Fp), hz(A, rows, Fp)
    Wh, Wl, ws, cc = hz(A, 128, Fp), hz(A, 128, Fp), z(A, 128), z(A, 128)
    _lib.check(lib.iplan_learner_row_stats(P(X), X.stride(0), Fp, F, rows, A, P(stat), st), "row_stats")
    _lib.check(lib.iplan_learner_x_split(P(X), X.numel(), P(Xh), P(Xl), st), "x_split")

    def timed(call):
        call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    Z = torch.full((A, rows, 128), float("nan"), device=dev)
    fwd = lambda: _lib.check(lib.iplan_learner_fc1_forward(
        P(actor.flat), actor.stride(), P(critic.flat), critic.stride(), P(Xh), P(Xl), Xh.stride(0), Fp, F, rows, A, P(stat),
        P(Wh), P(Wl), P(ws), P(cc), P(Z), st), "fc1_forward")
    t_fwd = timed(fwd)
    xs = X[..., :F].double()
    mu, var = xs.mean(-1, keepdim=True), xs.var(-1, unbiased=False, keepdim=True)
    xn = (xs - mu) / torch.sqrt(var + 1e-5)
    zr = torch.empty(A, rows, 128, dtype=torch.float64, device=dev)
    for a in range(A):
        for t, stack in enumerate((actor, critic)):
            sd = stack.nets[a].state_dict()
            y = xn[a] * sd["base.feature_norm.weight"].double() + sd["base.feature_norm.bias"].double()
            zr[a, :, 64 * t:64 * t + 64] = y @ sd["base.mlp.fc1.0.weight"].double().T + sd["base.mlp.fc1.0.bias"].double()
    d_fwd = (Z.double() - zr).abs().max().item() / zr.abs().max().item()
    # ---- backward: G = dZ1^T X ---------------------------------------------------------------------------
    dZ = torch.randn(A, rows, 128, device=dev) * 1e-3
    SM = torch.randn(A, 2, 128, device=dev) * 1e-3
    Dh, Dl, gs, G = hz(A, rows, 128), hz(A, rows, 128), z(2 * A), z(A, 128, Fp)
    ga, gc = torch.zeros_like(actor.flat), torch.zeros_like(critic.flat)
    bwd = lambda: _lib.check(lib.iplan_learner_fc1_backward(
        P(actor.flat), actor.stride(), P(critic.flat), critic.stride(), P(ga), P(gc), P(Xh), P(Xl), Xh.stride(0), Fp, F, rows, A,
        P(dZ), P(Dh), P(Dl), P(gs), P(SM), P(G), st), "fc1_backward")
    t_bwd = timed(bwd)
    Gref = torch.einsum("ark,arf->akf", dZ.double(), X.double())
    d_bwd = (G.double() - Gref).abs().max().item() / Gref.abs().max().item()
    print(f"A={A} rows={rows} F={F}: forward {t_fwd:.3f} ms, max rel|Z1 - fp64| = {d_fwd:.3e}; "
          f"backward (all launches) {t_bwd:.3f} ms, max rel|G - fp64| = {d_bwd:.3e}; "
          f"nan: {bool(torch.isnan(Z).any() or torch.isnan(G).any())}", flush=True)
    if kernel_rates:
        print(f"  {torch.cuda.get_device_name()}:")
        rates("forward (fc1_fwd_wgmma_kernel)", kernel_ms(fwd, "fc1_fwd_wgmma_kernel", 10), A, rows, Fp)
        rates("backward (fc1_bwd_wgmma_kernel)", kernel_ms(bwd, "fc1_bwd_wgmma_kernel", 10), A, rows, Fp)
    return max(d_fwd, d_bwd)


if __name__ == "__main__":
    ok = run(2, 300, 272) < 1e-5            # MPE width: ragged k (Fp = 288) and ragged rows
    ok &= run(1, 128, 2485) < 1e-5
    ok &= run(5, 46592, 2485, reps=3, kernel_rates=True) < 1e-5   # bench shape: 512 envs x 91 steps
    print("OK" if ok else "MISMATCH")
