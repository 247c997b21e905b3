"""`python bench.py --workload train`: BASELINE config 4 - one NeuMesh training step per GPU per iteration.

A step = 512 rays per GPU (`configs/neumesh_dtu_scan63.yaml` N_rays) of a synthetic spiral frame: fused no-grad sampling
cascade (perturb=True), differentiable field evaluation at the 128 + 127 final samples of every ray through
``FusedFieldFn`` (CUDA forward + backward, ``csrc/train.cu``), torch-op compositing and losses (image L1, eikonal on
``implicit_nablas``, mask BCE, indicator regulariser - ``models/trainer.py:173-262`` without the NeuS-teacher
distillation terms: the teacher is out of scope, DESIGN.md), backward, gradient all-reduce over NCCL (data parallel, as the
reference's DDP ``train.py:326-332``), Adam step.  Prints one JSON line: rays/s over all GPUs."""
from __future__ import annotations

import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_RAYS = 512
KW = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True, detailed_output=True, perturb=True)


def run_reference(args, world):
    """CPU arm of the training workload: the reference's training-step arithmetic (torch autograd through the generic
    renderer and the torch-op field, exact KNN by the oracle) on the host cores, on a bounded sample of rays per step."""
    import time
    import torch.nn.functional as F
    import bench
    import neumesh_b200 as nb
    from neumesh_b200 import synth
    from oracle.mesh_grid import OracleMeshGrid
    torch.set_num_threads(bench.host_cores())
    n = 64
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = nb.NeuMesh(OracleMeshGrid(mesh), **cfg.model_kwargs())
    model.load_state_dict(sd)
    model.train()
    model.fused_train = False            # plain torch autograd on the CPU: the reference's own arithmetic
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    normals0 = model.mesh_grid.get_vertex_normal_torch().detach().clone()
    g = torch.Generator().manual_seed(1234)

    def step(i):
        o, d = synth.frame_rays(800, 800, view=i % 90)
        sel = torch.randint(0, o.shape[0], (n,), generator=g)
        tgt, msk = torch.rand(n, 3, generator=g), (torch.rand(n, generator=g) > 0.5).float()
        opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o[sel], d[sel], model, rayschunk=4096, **KW)
        nab_norm = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        loss = F.l1_loss(rgb, tgt) + 0.1 * F.mse_loss(nab_norm, torch.ones_like(nab_norm)) \
            + 0.1 * F.binary_cross_entropy(acc, msk) + 0.01 * F.mse_loss(model.indicator_vector, normals0)
        loss.backward()
        opt.step()

    step(0)      # builds the kd-tree, warms MKL
    t = time.perf_counter()
    for i in range(args.steps):
        step(1 + i)
    dt = time.perf_counter() - t
    val = n * args.steps / dt
    print(json.dumps({
        "impl": "reference", "metric": "train_rays_per_sec_512_rays_per_gpu", "value": val, "unit": "rays/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
        "config": {"workload": "train_step_icosphere_V163842_F32_K8_512rays_per_gpu", "rays_per_step_sample": n},
        "cpu_baseline": {"value": val, "unit": "rays/s", "cores": bench.host_cores(), "kind": "port",
                         "sample": f"{n} rays per step (torch CPU autograd through the generic renderer + torch-op field, "
                                   f"oracle exact KNN), forward + backward + Adam"},
        "e2e": {"value": val, "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}), flush=True)


def main(args, rank, world, local_rank):
    import torch.distributed as dist
    import torch.nn.functional as F
    import bench
    import neumesh_b200 as nb
    from neumesh_b200 import _lib, synth

    if args.impl == "reference":
        if rank == 0:
            run_reference(args, world)
        return
    assert torch.cuda.is_available(), "bench needs a CUDA device"
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = nb.NeuMesh(nb.MeshGrid(mesh, dev), mlp_engine=args.engine, **cfg.model_kwargs())
    model.load_state_dict(sd)
    model = model.to(dev).train()
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    params = [p for p in model.parameters() if p.requires_grad]
    normals0 = model.mesh_grid.get_vertex_normal_torch().detach().clone()
    n_in = args.warmup + args.steps
    g = torch.Generator().manual_seed(1234 + rank)
    host = []
    for i in range(n_in):
        o, d = synth.frame_rays(800, 800, view=i % 90)
        sel = torch.randint(0, o.shape[0], (N_RAYS,), generator=g)
        tgt = torch.rand(N_RAYS, 3, generator=g)
        msk = (torch.rand(N_RAYS, generator=g) > 0.5).float()
        host.append(tuple(t.contiguous().pin_memory() for t in (o[sel], d[sel], tgt, msk)))

    def step(i):
        o, d, tgt, msk = (t.to(dev, non_blocking=True) for t in host[i % len(host)])
        opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, **KW)
        nab_norm = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        loss = F.l1_loss(rgb, tgt) + 0.1 * F.mse_loss(nab_norm, torch.ones_like(nab_norm)) \
            + 0.1 * F.binary_cross_entropy(acc, msk) + 0.01 * F.mse_loss(model.indicator_vector, normals0)
        loss.backward()
        if world > 1:   # data-parallel gradient all-reduce (dense: MLP weights and both vertex tables)
            flat = torch.cat([p.grad.reshape(-1) for p in params if p.grad is not None])
            dist.all_reduce(flat)
            flat /= world
            off = 0
            for p in params:
                if p.grad is not None:
                    n = p.grad.numel()
                    p.grad.copy_(flat[off:off + n].view_as(p.grad))
                    off += n
        opt.step()
        return loss

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # started before the warm-up: nvidia-smi's start-up stalls driver calls for a few hundred ms (bench.py)
    sampler = bench.ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
        sampler.wait_ready()
    for i in range(args.warmup):
        step(i)
    barrier()
    l0 = _lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    sampler.mark()
    e0.record()
    losses = []
    for i in range(args.steps):
        losses.append(step(args.warmup + i))
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    launches = _lib.launch_count() - l0
    clocks = sampler.stop() if rank == 0 else None
    # end to end: the same steps with the loss read back to the host every step
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    f0.record()
    for i in range(args.steps):
        float(step(args.warmup + i).item())
    f1.record()
    barrier()
    ms2 = torch.tensor([f0.elapsed_time(f1)], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        dist.all_reduce(ms2, op=dist.ReduceOp.MAX)
    if rank == 0:
        rays = N_RAYS * world * args.steps
        pts = N_RAYS * 255
        flop_fwd = N_RAYS * (255 * (bench.FLOP_GEO + bench.FLOP_JVP) + 127 * bench.FLOP_COL)
        line = {"metric": "train_rays_per_sec_512_rays_per_gpu", "value": rays / (ms.item() * 1e-3), "unit": "rays/s",
                "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms.item() / args.steps,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "fp32 (training kernels: fp32 FFMA; sampling cascade: fp16x3 / 3xTF32 wgmma)",
                "data": "synthetic",
                "config": {"workload": "train_step_icosphere_V163842_F32_K8_512rays_per_gpu", "rays_per_gpu": N_RAYS,
                           "points_per_gpu_per_step": pts, "render": KW, "optimizer": "Adam",
                           "losses": "img L1 + 0.1 eikonal + 0.1 mask BCE + 0.01 indicator reg (no NeuS-teacher terms)",
                           "parallelism": f"data parallel x{world}, dense gradient all-reduce",
                           "l2": "every step renders rays of a different spiral view; activations of a step (~2.4 GB) "
                                 "exceed the 126 MB L2"},
                "e2e": {"value": rays / (ms2.item() * 1e-3), "unit": "rays/s", "ms_per_step": ms2.item() / args.steps,
                        "h2d_bytes_per_step": N_RAYS * 10 * 4, "d2h_bytes_per_step": 4,
                        "api": "neumesh_b200.volume_render under autograd on pinned host rays + backward + Adam; loss "
                               "read back every step"},
                "gpu_launches": int(launches), "clocks": clocks,
                "roofline": {"bound": "fp32", "kernel": "nmb::tr::sgemm_kernel (training GEMMs) + per-point kernels",
                             "achieved": 3.0 * flop_fwd / (ms.item() / args.steps * 1e-3) / 1e12, "peak": None,
                             "unit": "TFLOP/s", "frac": None, "traffic": None,
                             "note": "achieved = 3 x forward algorithmic FLOPs (forward + data and weight gradients) / "
                                     "WHOLE step time (includes sampling cascade, compositing, all-reduce, Adam)"},
                "final_loss": float(losses[-1].item())}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
