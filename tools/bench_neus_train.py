#!/usr/bin/env python
"""The NeuS stage-1 training step (``configs/neus_dtu_scan63.yaml``) on its three routes, side by side:

* ``torch``: the torch-op path (``fused_train = False``): autograd nabla with ``create_graph=True``, double backward;
* ``fused_fp32``: ``neus_ops.FusedSurfaceFn`` / ``FusedRadianceFn`` on ``nmb_tr_gemm`` (the default route);
* ``fused_tf32x3``: the same ops on ``nmb_tr_gemm_tc`` (3xTF32 on the tensor cores).

    python tools/bench_neus_train.py [--rounds 5] [--steps 10] [--warmup 3] [--out result.json]

The step: 512 rays of a synthetic frame, ``nb.volume_render`` with the config's render settings (64 + 4 x 16 samples,
calc_normal, perturb, unbounded near/far), image L1 over the masked rays + mask BCE + 0.1 eikonal as
``models/trainer.py`` computes them, Adam at 5e-4, all from fixed seeds.  The arms alternate in rounds (CUDA events,
median ms per step over the rounds); peak memory is ``torch.cuda.max_memory_allocated`` over each arm's timed steps;
the 20-step loss trajectories of the three arms start from the same parameters and batches.  The card's name, power
limit and maximum SM clock are read with nvidia-smi in the same run.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neumesh_b200 as nb  # noqa: E402
from neumesh_b200 import synth  # noqa: E402

N_RAYS = 512
NEUS_KW = dict(variance_init=0.05, speed_factor=10.0, W_geo_feat=256, obj_bounding_radius=1.0,
               surface_cfg=dict(embed_multires=6, radius_init=0.5, geometric_init=True, D=8, W=256, skips=[4]),
               radiance_cfg=dict(embed_multires=-1, embed_multires_view=4, use_view_dirs=True, D=4, W=256, skips=[]))
RENDER_KW = dict(calc_normal=True, white_bkgd=False, bounded_near_far=False, detailed_output=True, perturb=True,
                 N_samples=64, N_importance=64, N_upsample_iters=4, obj_bounding_radius=1.0)
ARMS = {"torch": (False, "fp32"), "fused_fp32": (True, "fp32"), "fused_tf32x3": (True, "tf32x3")}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def batches(n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        o, d = synth.frame_rays(800, 800, view=i % 90)
        sel = torch.randint(0, o.shape[0], (N_RAYS,), generator=g)
        tgt, msk = torch.rand(N_RAYS, 3, generator=g), torch.rand(N_RAYS, generator=g) > 0.5
        out.append(tuple(t.contiguous().pin_memory() for t in (o[sel], d[sel], tgt, msk)))
    return out


class Arm:
    def __init__(self, name, dev, seed=0):
        fused, engine = ARMS[name]
        torch.manual_seed(seed)
        self.model = nb.NeuS(train_engine=engine, **NEUS_KW).to(dev).train()
        self.model.fused_train = fused
        self.opt = torch.optim.Adam(self.model.parameters(), lr=5e-4)
        self.dev = dev

    def step(self, batch, seed):
        o, d, tgt, msk = (t.to(self.dev, non_blocking=True) for t in batch)
        torch.manual_seed(seed)        # the perturbation draws: the same for every arm
        self.opt.zero_grad(set_to_none=True)
        rgb, _, ex = nb.volume_render(o, d, self.model, rayschunk=4096, **RENDER_KW)
        nab = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        m = msk.float()
        l_img = (F.l1_loss(rgb, tgt, reduction="none") * m[..., None]).sum() / (m.sum() + 1e-10)
        loss = l_img + F.binary_cross_entropy(acc, m) + 0.1 * F.mse_loss(nab, torch.ones_like(nab))
        loss.backward()
        self.opt.step()
        return loss


def step_times(dev, rounds, steps, warmup):
    arms = {k: Arm(k, dev) for k in ARMS}
    data = batches(warmup + steps, seed=1234)
    for a in arms.values():
        for i in range(warmup):
            a.step(data[i], i)
    per, peak = {k: [] for k in arms}, {k: 0 for k in arms}
    names = list(arms)
    for r in range(rounds):
        for k in (names if r % 2 == 0 else names[::-1]):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(steps):
                arms[k].step(data[warmup + i], warmup + i)
            b.record()
            b.synchronize()
            per[k].append(a.elapsed_time(b) / steps)
            peak[k] = max(peak[k], torch.cuda.max_memory_allocated(dev))
    return {k: {"median_ms_per_step": statistics.median(per[k]), "rounds_ms": per[k],
                "max_memory_allocated_MiB": peak[k] / 2 ** 20} for k in arms}


def loss_trajectories(dev, steps=20):
    data = batches(steps, seed=4321)
    traj = {}
    for k in ARMS:
        arm = Arm(k, dev)
        traj[k] = [float(arm.step(data[i], i)) for i in range(steps)]
        del arm
    drift = {k: max(abs(a - b) / abs(b) for a, b in zip(traj[k], traj["torch"])) for k in ARMS if k != "torch"}
    return {"loss": traj, "max_relative_difference_to_torch": drift}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    res = {"gpu_before": gpu_info()}
    res["step"] = step_times(dev, args.rounds, args.steps, args.warmup)
    t = res["step"]["torch"]["median_ms_per_step"]
    for k in ("fused_fp32", "fused_tf32x3"):
        res["step"][k]["speedup_vs_torch"] = t / res["step"][k]["median_ms_per_step"]
    res["loss_trajectories"] = loss_trajectories(dev)
    res["gpu_after"] = gpu_info()   # name, power limit, max SM clock
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
