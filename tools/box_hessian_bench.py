"""Timing of the masked passes behind LBFGSBSolver's final_approx_free_* members (DESIGN.md §8g), with the card's name and power limit
read in the same run.

For n in {1e6, 1e7}, m = c in {10, 20} (fp64, random pairs, half the rows free at random) and k in {1, 4, 16}, CUDA events on the
context's stream, best of three windows of R calls each:
  - the product B_F V or H_F V as BFGSMat runs it: lbfgs_b200_hist_wt_dot_multi_masked, then lbfgs_b200_hist_lincomb_multi_masked
    (the 2c x 2c algebra between them is host work and is left out: the coefficients are fixed);
  - the unfused route on the same data: V zeroed off F (a torch multiply on the same stream), the unmasked hist_wt_dot_multi and
    hist_lincomb_multi, and OUT zeroed off F;
  - the diagonal: lbfgs_b200_hist_quad_diag_masked against hist_quad_diag followed by zeroing off F;
  - the masked Gram pass (lbfgs_b200_hist_masked_gram), which the H_F members run once per free set (BFGSMat keeps its result).
GB/s on the traffic model, w = 8 bytes per element, one class byte per row for the masked passes:
      masked dots  w n (2c + k) + n        masked combination  w n (2c + 2k) + n        masked diagonal  w n (2c + 1) + n
      unfused      the unmasked passes' w n (2c + k) + w n (2c + 2k), plus 3 w n k to zero V and OUT (read V and a mask, write)

Usage: python tools/box_hessian_bench.py [--reps R] [--out FILE]   (one JSON object on stdout; FILE also receives it)
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch   # before lbfgspp_b200: both load NCCL, and torch needs its own build of it

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402
from tools.hessian_sample_bench import card  # noqa: E402


class TorchArray:
    """A torch tensor as the History methods take a DeviceArray (they read .ptr only)."""

    def __init__(self, t):
        self.t, self.ptr = t, C.c_void_p(t.data_ptr())


def best_ms(ctx, fn, reps):
    fn()
    ctx.sync()
    best = float("inf")
    for _ in range(3):
        ctx.timer_start()
        for _ in range(reps):
            fn()
        best = min(best, ctx.timer_stop() / reps)
    return best


def run(ctx, reps):
    stream = torch.cuda.ExternalStream(ctx.lib.lbfgs_b200_stream(ctx.h))   # torch's zeroing on the context's stream, so events bracket all
    w, out = 8, []
    for n in (1_000_000, 10_000_000):
        rng = np.random.default_rng(n)
        F = rng.random(n) < 0.5
        cls = np.where(F, lb.CLS_FINAL, 0).astype(np.uint8)
        maskf = torch.tensor(F.astype(np.float64), device="cuda")
        for m in (10, 20):
            h = lb.History(ctx, n, m)
            for _ in range(m):
                s = rng.standard_normal(n)
                h.add(ctx.array(s), ctx.array(s * (1.0 + rng.random(n))))
            box = lb.Box(h)
            box.set("cls", cls)
            c = h.ncorr
            K = rng.standard_normal((2 * c, 2 * c))
            K = K + K.T
            d = ctx.empty(n)
            with torch.cuda.stream(stream):
                dt = torch.empty(n, dtype=torch.float64, device="cuda")
                diag = TorchArray(dt)
                t_dm = best_ms(ctx, lambda: h.quad_diag_masked(box, lb.CLS_FINAL, 2.0, K, d), reps)
                t_du = best_ms(ctx, lambda: (h.quad_diag(2.0, K, diag), dt.mul_(maskf)), reps)
                out.append(dict(n=n, m=m, k=None, op="diagonal", masked_ms=t_dm, unfused_ms=t_du,
                                masked_GBps=(w * n * (2 * c + 1) + n) / t_dm / 1e6))
                G = (C.c_double * (4 * c * c))()
                gram = getattr(ctx.lib, "lbfgs_b200_hist_masked_gram_f64")
                t_g = best_ms(ctx, lambda: ctx.check(gram(h.h, box.h, box._ptr("cls"), lb.CLS_FINAL, G)), reps)
                out.append(dict(n=n, m=m, k=None, op="masked_gram", masked_ms=t_g, masked_GBps=(w * n * 2 * c + n) / t_g / 1e6))
                for k in (1, 4, 16):
                    Vt = torch.tensor(rng.standard_normal(k * n), device="cuda")
                    Vz, Ot = torch.empty_like(Vt), torch.empty_like(Vt)
                    V, VZ, O = TorchArray(Vt), TorchArray(Vz), TorchArray(Ot)
                    Cc = rng.standard_normal((2 * c, k))
                    t_dots = best_ms(ctx, lambda: h.wt_dot_multi_masked(box, lb.CLS_FINAL, V, k, n), reps)
                    t_comb = best_ms(ctx, lambda: h.lincomb_multi_masked(box, lb.CLS_FINAL, 0.5, V, k, n, Cc, O, n), reps)

                    def unfused():
                        torch.mul(Vt.view(k, n), maskf, out=Vz.view(k, n))
                        h.wt_dot_multi(VZ, k, n)
                        h.lincomb_multi(0.5, VZ, k, n, Cc, O, n)
                        Ot.view(k, n).mul_(maskf)

                    t_unf = best_ms(ctx, unfused, reps)
                    out.append(dict(n=n, m=m, k=k, op="product", masked_dots_ms=t_dots, masked_comb_ms=t_comb, masked_ms=t_dots + t_comb,
                                    unfused_ms=t_unf, masked_dots_GBps=(w * n * (2 * c + k) + n) / t_dots / 1e6,
                                    masked_comb_GBps=(w * n * (2 * c + 2 * k) + n) / t_comb / 1e6,
                                    unfused_GBps=(w * n * (4 * c + 3 * k) + 3 * w * n * k) / t_unf / 1e6))
            del box, h
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, power = card()
    ctx = lb.Context(0)
    res = dict(card=name, power_limit=power, results=run(ctx, a.reps))
    ctx.close()
    text = json.dumps(res)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
