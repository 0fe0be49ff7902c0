#!/usr/bin/env python3
"""Refine converted gaussians against views of their mesh with the standard 3DGS render's backward pass, and measure the
result on held-out views.

For each R: convert the bench scene (synth.helmet_standin(2048)) to PACKED56; render the mesh's albedo (m2s_mesh_render)
from `--train` training views and `--held` held-out views on an orbit around the model; replace the non-finite opacity
logits (the conversion writes +inf for alpha = 1) by a stated finite start, logit(0.99); run Adam with graphdeco's
per-field learning rates (position 1.6e-4 times the scene extent, rotation 1e-3, log-scale 5e-3, SH0 2.5e-3, opacity
logit 5e-2; eps 1e-15) on an L1 loss over RGBA against the albedo target, one training view per iteration in turn.
Reports m2s_image_compare's PSNR and SSIM (all pixels and covered pixels, both albedo and 3DGS alpha as covers) of the
3DGS RGBA8 image against the held-out albedo, averaged over the held-out views: as converted, after the finite start
(so the start is not credited to the fit), and after the fit; plus the ms per iteration of the forward pass and of the
backward pass (CUDA events).  `--ply-dir` writes the refined gaussians as standard .ply files there.  Prints one JSON
document with the card's name and power limit; `--out` also writes it to a file."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gs3d_bench import card  # noqa: E402
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402
from mesh2splat_b200 import _abi, synth  # noqa: E402
from mesh2splat_b200.api import Context, write_3dgs_ply  # noqa: E402

NEAR = 0.01
RADIUS = 3.2
LOGIT_START = math.log(0.99 / 0.01)   # the finite start of an infinite logit: opacity 0.99


def orbit(k: int, n: int, phase: float, w: int, h: int):
    """view k of n on the orbit: azimuth 2 pi (k + phase) / n, elevation alternating +-0.35 rad"""
    az = 2 * math.pi * (k + phase) / n
    el = 0.35 if k % 2 == 0 else -0.2
    eye = np.array([RADIUS * math.cos(el) * math.sin(az), RADIUS * math.sin(el), RADIUS * math.cos(el) * math.cos(az)])
    V = column_major(look_at(eye, np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(60.0), w / h, NEAR, 100.0))
    return V, P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="128,512,2048")
    ap.add_argument("--train", type=int, default=8)
    ap.add_argument("--held", type=int, default=4)
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=540)
    ap.add_argument("--lr-scale", type=float, default=1.0, help="every learning rate times this")
    ap.add_argument("--ply-dir")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    w, h = args.width, args.height
    M = column_major(np.eye(4, dtype=np.float32))
    res = {"card": card(), "width": w, "height": h, "train_views": args.train, "held_views": args.held, "iters": args.iters,
           "logit_start": LOGIT_START, "lr_scale": args.lr_scale, "runs": []}
    scene = synth.helmet_standin(2048)
    with Context(0) as ctx, ctx.gs3d_state() as state:
        ds = ctx.upload(scene)

        def views(n, phase):
            out = []
            for k in range(n):
                V, P = orbit(k, n, phase, w, h)
                alb = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
                ctx.mesh_render(ds, V, P, M, w, h, (NEAR, 100.0), 0, targets=("albedo",), gbuffer={"albedo": alb})
                out.append((V, P, alb, alb.view(h, w, 4).float() / 255.0))
            return out

        train, held = views(args.train, 0.0), views(args.held, 0.5)

        def score(prm):
            acc = {}
            for V, P, alb, _ in held:
                imgs, _, _ = ctx.render_3dgs(prm.detach().contiguous().view(-1).view(torch.uint8), prm.shape[0], _abi.LAYOUT_PACKED56,
                                             V, P, M, w, h, near=NEAR, targets=("rgba8",))
                r = ctx.compare_images(alb, imgs["rgba8"], w, h, alb, imgs["rgba8"])
                for k in ("psnr", "ssim", "psnr_covered", "ssim_covered"):
                    acc[k] = acc.get(k, 0.0) + r[k] / len(held)
            return acc

        for R in [int(x) for x in args.res.split(",")]:
            out = ctx.convert(ds, R, _abi.LAYOUT_PACKED56)
            n = out.written
            prm = out.data[: n * 56].view(torch.float32).view(n, 14).clone()
            row = {"R": R, "gaussians": n, "as_converted": score(prm)}
            bad = ~torch.isfinite(prm[:, 13])
            row["non_finite_logits"] = int(bad.sum())
            prm[bad, 13] = LOGIT_START
            row["finite_start"] = score(prm)
            leaves = [prm[:, a:b].clone().requires_grad_(True) for a, b in ((0, 3), (3, 7), (7, 10), (10, 13), (13, 14))]
            lrs = tuple(args.lr_scale * lr for lr in (1.6e-4 * RADIUS * 1.1, 1e-3, 5e-3, 2.5e-3, 5e-2))
            opt = torch.optim.Adam([{"params": [x], "lr": lr} for x, lr in zip(leaves, lrs)], eps=1e-15)
            fwd_ms, bwd_ms, losses = [], [], []
            for it in range(args.iters):
                V, P, _, target = train[it % len(train)]
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                opt.zero_grad()
                x = torch.cat(leaves, 1)
                e0.record()
                img = ctx.render_3dgs_grad(x, state, V, P, M, w, h, near=NEAR)
                e1.record()
                loss = (img - target).abs().mean()
                loss.backward()
                e2.record()
                opt.step()
                torch.cuda.synchronize()
                fwd_ms.append(e0.elapsed_time(e1))
                bwd_ms.append(e1.elapsed_time(e2))
                losses.append(float(loss.detach()))
            refined = torch.cat([x.detach() for x in leaves], 1)
            row["non_finite_after"] = int((~torch.isfinite(refined)).any(1).sum())
            row["refined"] = score(refined)
            row["train_l1_first_last"] = [float(np.mean(losses[: len(train)])), float(np.mean(losses[-len(train):]))]
            row["train_l1_curve"] = [float(np.mean(losses[i: i + len(train)])) for i in range(0, len(losses), max(len(train), len(losses) // 8))]
            row["forward_ms_per_iter"] = float(np.median(fwd_ms[len(train):]))
            row["backward_ms_per_iter"] = float(np.median(bwd_ms[len(train):]))
            if args.ply_dir:
                path = os.path.join(args.ply_dir, f"refined_R{R}.ply")
                write_3dgs_ply(path, refined)
                row["ply"] = path
            print(json.dumps(row), flush=True)
            res["runs"].append(row)
            del out, prm, leaves, opt, refined
            torch.cuda.empty_cache()
        ds.free()
    doc = json.dumps(res, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
