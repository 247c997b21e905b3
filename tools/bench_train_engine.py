#!/usr/bin/env python
"""The two GEMM engines of the training path side by side: ``train_engine="fp32"`` (``nmb_tr_gemm``, FFMA SGEMM) and
``"tf32x3"`` (``nmb_tr_gemm_tc``, 3xTF32 on wgmma).

    python tools/bench_train_engine.py [--rounds 5] [--steps 20] [--out result.json]

1. The training step of ``bench_train.py`` (512 rays, V = 163 842 icosphere, calc_normal, perturb, Adam), without and
   with the NeuS teacher and the distillation losses of ``examples/train_distill.py``: both engines alternating, rounds x
   steps after warm-up, CUDA events; the median ms per step over the rounds.
2. A ``torch.profiler`` run (CUDA activities) of the step with the teacher per engine: GEMM kernel time and its share of
   the step's kernel time.
3. Per production GEMM shape, both engines: kernel time by CUDA events over repeated launches (split-K products include
   their reduction kernel) and achieved TFLOP/s = 2 M N K / time.  Ceilings (H100 SXM data sheet, dense, 700 W):
   FP32 67 TFLOP/s for the SGEMM; TF32 495 TFLOP/s, i.e. 165 TFLOP/s of 3xTF32 products (three MMAs per product).
4. The 20-step loss trajectories of both engines from the same seeds and their relative difference.

The card's name, power limit and maximum SM clock are read with nvidia-smi in the same run and printed beside the
numbers."""
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
from neumesh_b200 import synth, train_ops  # noqa: E402

N_RAYS = 512
ENGINES = ("fp32", "tf32x3")
KW = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True, detailed_output=True, perturb=True)
TEACHER_KW = dict(variance_init=0.05, speed_factor=10.0, W_geo_feat=256, obj_bounding_radius=1.0,
                  surface_cfg=dict(embed_multires=6, radius_init=0.5, geometric_init=True, D=8, W=256, skips=[4]),
                  radiance_cfg=dict(embed_multires=-1, embed_multires_view=4, use_view_dirs=True, D=4, W=256, skips=[]))
GEMM_KERNELS = {"fp32": ("sgemm_kernel",), "tf32x3": ("gemm_tf32x3_kernel",)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


class Trainer:
    """A student (and its optimiser) on one engine; the teacher is shared and frozen."""

    def __init__(self, mesh, cfg, sd, engine, dev, teacher):
        self.model = nb.NeuMesh(nb.MeshGrid(mesh, dev), train_engine=engine, **cfg.model_kwargs())
        self.model.load_state_dict(sd)
        self.model = self.model.to(dev).train()
        self.opt = torch.optim.Adam(self.model.parameters(), lr=5e-4)
        self.normals0 = self.model.mesh_grid.get_vertex_normal_torch().detach().clone()
        self.teacher, self.engine, self.dev = teacher, engine, dev

    def step(self, batch, with_teacher):
        o, d, tgt, msk = (t.to(self.dev, non_blocking=True) for t in batch)
        self.opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o, d, self.model, rayschunk=4096, samples_output=with_teacher, **KW)
        nab = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        loss = F.l1_loss(rgb, tgt) + 0.1 * F.mse_loss(nab, torch.ones_like(nab)) \
            + 0.1 * F.binary_cross_entropy(acc, msk) + 0.01 * F.mse_loss(self.model.indicator_vector, self.normals0)
        if with_teacher:
            self.teacher.train_engine = self.engine
            with torch.no_grad():
                gt_sdf, gt_rad = self.teacher(ex["xyz"], ex["dirs"])
            loss = loss + 0.5 * F.l1_loss(ex["density"], gt_sdf.unsqueeze(-1)) + 0.5 * F.mse_loss(ex["colors"], gt_rad)
        loss.backward()
        self.opt.step()
        return loss


def batches(n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        o, d = synth.frame_rays(800, 800, view=i % 90)
        sel = torch.randint(0, o.shape[0], (N_RAYS,), generator=g)
        tgt, msk = torch.rand(N_RAYS, 3, generator=g), (torch.rand(N_RAYS, generator=g) > 0.5).float()
        out.append(tuple(t.contiguous().pin_memory() for t in (o[sel], d[sel], tgt, msk)))
    return out


def make_teacher(dev):
    torch.manual_seed(0)
    return nb.NeuS(**TEACHER_KW).to(dev).eval()


def step_times(mesh, cfg, sd, dev, rounds, steps, warmup):
    teacher = make_teacher(dev)
    tr = {e: Trainer(mesh, cfg, sd, e, dev, teacher) for e in ENGINES}
    data = batches(warmup + steps, seed=1234)
    res = {}
    for with_teacher in (False, True):
        variant = "with_teacher" if with_teacher else "student_only"
        for e in ENGINES:
            for i in range(warmup):
                tr[e].step(data[i], with_teacher)
        per = {e: [] for e in ENGINES}
        for r in range(rounds):
            for e in (ENGINES if r % 2 == 0 else ENGINES[::-1]):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(steps):
                    tr[e].step(data[warmup + i], with_teacher)
                b.record()
                b.synchronize()
                per[e].append(a.elapsed_time(b) / steps)
        res[variant] = {e: {"median_ms_per_step": statistics.median(per[e]), "rounds_ms": per[e]} for e in ENGINES}
        res[variant]["speedup"] = res[variant]["fp32"]["median_ms_per_step"] / res[variant]["tf32x3"]["median_ms_per_step"]
    return res


def profile_steps(mesh, cfg, sd, dev, n_steps=3):
    from torch.profiler import ProfilerActivity, profile
    teacher = make_teacher(dev)
    data = batches(n_steps + 2, seed=99)
    out = {}
    for e in ENGINES:
        t = Trainer(mesh, cfg, sd, e, dev, teacher)
        for i in range(2):
            t.step(data[i], True)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(n_steps):
                t.step(data[2 + i], True)
            torch.cuda.synchronize()
        total = gemm = red = 0.0
        for ev in prof.key_averages():
            us = ev.self_device_time_total      # device time of the kernels (runtime API entries carry none)
            if any(k in ev.key for k in GEMM_KERNELS[e]):
                gemm += us
            elif "reduce_splits" in ev.key:
                red += us
            total += us
        out[e] = {"gemm_ms_per_step": gemm / 1e3 / n_steps, "split_reduce_ms_per_step": red / 1e3 / n_steps,
                  "kernel_ms_per_step": total / 1e3 / n_steps, "gemm_share_of_kernel_time": gemm / max(total, 1e-9)}
    return out


def gemm_shapes(cfg):
    c = cfg.model_kwargs()
    spec = train_ops.FieldSpec(c["geometry_dim"], c["color_dim"], c["multires_d"], c["multires_fg"], c["multires_ft"],
                               c["multires_view"], c["enable_nablas_input"], c["D_density"], c["D_color"])
    M, Mt = N_RAYS * 255, 4 * N_RAYS * 127
    # (name, M, N, K, a_kcontig, b_kcontig, bias)
    return [
        (f"forward X.W^T K={spec.Kg}", M, 256, spec.Kg, True, True, True),
        ("forward X.W^T K=256", M, 256, 256, True, True, True),
        (f"forward X.W^T K={spec.Kc}", M, 256, spec.Kc, True, True, True),
        (f"forward tangent seed K={spec.chd}", M, 256, spec.chd, True, True, False),
        ("backward data dZ.W N=256", M, 256, 256, True, False, False),
        (f"backward data dZ.W N={spec.Kg}", M, spec.Kg, 256, True, False, False),
        (f"backward data dZ.W N={spec.chd}", M, spec.chd, 256, True, False, False),
        ("weight gradient dZ^T.X 256x256", 256, 256, M, False, False, False),
        (f"weight gradient dZ^T.X 256x{spec.Kg}", 256, spec.Kg, M, False, False, False),
        (f"weight gradient dZ^T.X 256x{spec.chd}", 256, spec.chd, M, False, False, False),
        ("NeuS teacher 4M x 256, K=256", Mt, 256, 256, True, True, False),
    ]


def gemm_times(cfg, dev, reps=20):
    out = []
    for (name, M, N, K, akc, bkc, use_bias) in gemm_shapes(cfg):
        A = torch.randn(M * K, device=dev)
        B = torch.randn(N * K, device=dev)
        C = torch.empty(M, N, device=dev)
        bias = torch.randn(N, device=dev) if use_bias else None
        row = {"shape": name, "M": M, "N": N, "K": K}
        for e in ENGINES:
            P = train_ops.CudaPrims(dev, e)
            call = lambda: P.gemm(A, K if akc else M, akc, B, K if bkc else N, bkc, C, N, M, N, K, bias=bias)  # noqa
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                call()
            b.record()
            b.synchronize()
            ms = a.elapsed_time(b) / reps
            row[e] = {"ms": ms, "tflops": 2.0 * M * N * K / ms / 1e9}
        row["speedup"] = row["fp32"]["ms"] / row["tf32x3"]["ms"]
        out.append(row)
    return out


def loss_trajectories(mesh, cfg, sd, dev, steps=20):
    data = batches(steps, seed=4321)
    traj = {}
    for e in ENGINES:
        teacher = make_teacher(dev)
        t = Trainer(mesh, cfg, sd, e, dev, teacher)
        traj[e] = [float(t.step(data[i], True)) for i in range(steps)]
    rel = [abs(a - b) / abs(a) for a, b in zip(traj["fp32"], traj["tf32x3"])]
    return {"loss": traj, "relative_difference": rel, "max_relative_difference": max(rel)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    res = {"gpu": gpu_info()}
    print("gpu (name, power limit, max SM clock):", res["gpu"], flush=True)
    res["gemm_shapes"] = gemm_times(cfg, dev)
    for r in res["gemm_shapes"]:
        print(f"{r['shape']:38s} fp32 {r['fp32']['ms']:7.3f} ms {r['fp32']['tflops']:6.1f} TFLOP/s | tf32x3 "
              f"{r['tf32x3']['ms']:7.3f} ms {r['tf32x3']['tflops']:6.1f} TFLOP/s | x{r['speedup']:.2f}", flush=True)
    res["step"] = step_times(mesh, cfg, sd, dev, args.rounds, args.steps, args.warmup)
    for v in ("student_only", "with_teacher"):
        s = res["step"][v]
        print(f"step {v:13s}: fp32 {s['fp32']['median_ms_per_step']:.2f} ms, tf32x3 "
              f"{s['tf32x3']['median_ms_per_step']:.2f} ms (x{s['speedup']:.2f}); rounds fp32 "
              f"{[round(x, 2) for x in s['fp32']['rounds_ms']]} tf32x3 {[round(x, 2) for x in s['tf32x3']['rounds_ms']]}",
              flush=True)
    res["profile_with_teacher"] = profile_steps(mesh, cfg, sd, dev)
    for e, p in res["profile_with_teacher"].items():
        print(f"profile {e}: GEMM {p['gemm_ms_per_step']:.2f} ms + split reduce {p['split_reduce_ms_per_step']:.2f} ms "
              f"of {p['kernel_ms_per_step']:.2f} ms kernel time per step ({100 * p['gemm_share_of_kernel_time']:.1f} %)",
              flush=True)
    res["loss_trajectories"] = loss_trajectories(mesh, cfg, sd, dev)
    lt = res["loss_trajectories"]
    print("loss fp32  :", [round(x, 5) for x in lt["loss"]["fp32"]])
    print("loss tf32x3:", [round(x, 5) for x in lt["loss"]["tf32x3"]])
    print(f"max relative loss difference over 20 steps: {lt['max_relative_difference']:.2e}")
    print("gpu (name, power limit, max SM clock):", gpu_info(), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
