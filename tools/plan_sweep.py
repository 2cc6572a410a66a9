#!/usr/bin/env python
"""Planner sweep for forward / data-gradient GEMMs: for each listed shape, times the planner's own choice and every forced
(wgmma N, split-K) combination (T2V_FORCE_BN / T2V_FORCE_FWD_SPLITS), L2-cold (rotating
operand sets), CUDA-graph replay, CUDA events.  The CSV lines are what the fwd / dgrad cost model in csrc/gemm_plan.cu
(fwd_cost) is fitted to; cuBLAS on the same shape is printed as the yardstick.
  python tools/plan_sweep.py > gpurun_out/plan_sweep.txt"""
import itertools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from cublas_compare import time_graph  # noqa: E402
from t2v_b200 import prims  # noqa: E402

# (N, H, W, Cin, Cout, KH, KW): linear layers as 1x1 on a [1,1,M] image, convolutions as they appear in cfg 2
SHAPES = [
    (1, 1, 1024, 1280, 1280, 1, 1), (1, 1, 1024, 1280, 3840, 1, 1), (1, 1, 1024, 1280, 10240, 1, 1), (1, 1, 1024, 5120, 1280, 1, 1),
    (1, 1, 4096, 640, 640, 1, 1), (1, 1, 4096, 640, 1920, 1, 1), (1, 1, 4096, 640, 5120, 1, 1), (1, 1, 4096, 2560, 640, 1, 1),
    (1, 1, 16384, 320, 320, 1, 1), (1, 1, 16384, 320, 2560, 1, 1), (1, 1, 16384, 1280, 320, 1, 1),
    (16, 8, 8, 1280, 1280, 3, 3), (16, 16, 16, 640, 640, 3, 3), (16, 4, 4, 1280, 1280, 3, 3), (16, 8, 8, 2560, 1280, 3, 3),
    (1, 16, 64, 1280, 1280, 3, 1), (1, 16, 256, 640, 640, 3, 1), (1, 16, 16, 1280, 1280, 3, 1),
]
ENV = ("T2V_FORCE_BN", "T2V_FORCE_FWD_SPLITS")


def main():
    dev = torch.device("cuda", 0)
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    for shp in SHAPES:
        N, H, W, Ci, Co, KH, KW = shp
        pads = ((KH - 1) // 2, (KH - 1) // 2, (KW - 1) // 2, (KW - 1) // 2)
        M = N * H * W
        per = 2 * (M * Ci + Co * KH * KW * Ci + M * Co)
        nset = min(16, max(4, -(-(300 << 20) // per)))
        reps = max(8, nset)
        xs = [torch.randn(N, H, W, Ci, device=dev).bfloat16() for _ in range(nset)]
        ws = [(torch.randn(Co, KH, KW, Ci, device=dev) * 0.02).bfloat16() for _ in range(nset)]
        dys = [torch.randn(N, H, W, Co, device=dev).bfloat16() for _ in range(nset)]
        bias = torch.randn(Co, device=dev)
        fl = 2.0 * M * Co * KH * KW * Ci
        forms = {"fwd": [lambda i=i: prims.conv_fwd(xs[i], ws[i], bias, None, None, 1, pads) for i in range(nset)],
                 "dgrad": [lambda i=i: prims.conv_dgrad(dys[i], ws[i], (H, W), 1, pads) for i in range(nset)]}
        cub = None
        if KH == 1 and KW == 1:
            oy = [torch.empty(M, Co, device=dev, dtype=torch.bfloat16) for _ in range(nset)]
            cub = time_graph([lambda i=i: torch.mm(xs[i].view(M, Ci), ws[i].view(Co, Ci).t(), out=oy[i]) for i in range(nset)], reps)
        for kind, fns in forms.items():
            if only and only != kind:
                continue
            for k in ENV:
                os.environ.pop(k, None)
            base = time_graph(fns, reps)
            ncols = Co if kind == "fwd" else Ci
            kb = ((Ci if kind == "fwd" else Co) + 63) // 64 * KH * KW
            bns = sorted({b for b in (64, 96, 128) if b - 16 < ncols})
            rows = []
            for bn, mh, sp in itertools.product(bns, (1,), (1, 2, 3, 4, 6, 8)):
                if sp > 1 and (kb < 2 * sp):
                    continue
                os.environ["T2V_FORCE_BN"], os.environ["T2V_FORCE_FWD_SPLITS"] = str(bn), str(sp)
                try:
                    us = time_graph(fns, reps)
                except Exception as ex:  # noqa: BLE001
                    torch.cuda.synchronize()
                    print("ERR", kind, shp, bn, mh, sp, repr(ex)[:80])
                    continue
                rows.append((us, bn, mh, sp))
                print(f"CSV,{kind},{','.join(str(v) for v in shp)},{bn},{mh},{sp},{us:.2f}")
            for k in ENV:
                os.environ.pop(k, None)
            rows.sort()
            best = rows[0]
            cb = f"  cuBLAS {cub:.1f} us" if (cub and kind == "fwd") else ""
            print(f"{kind:5s} {shp}: planner {base:6.1f} us ({fl / base / 1e6:6.1f} TF/s) | best bn={best[1]} mh={best[2]} s={best[3]}: {best[0]:6.1f} us "
                  f"({fl / best[0] / 1e6:6.1f} TF/s)  gain {base / best[0]:.2f}x{cb}", flush=True)
        del xs, ws, dys
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
