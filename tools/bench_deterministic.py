"""Cost of ``torch.use_deterministic_algorithms(True)`` on the training step (bench_train.py's workload: V = 163 842
icosphere, 512 rays, perturb=True, image + eikonal + mask + indicator losses, Adam) on one GPU.

The two modes are timed alternately, ``--rounds`` windows of ``--steps`` steps each (CUDA events around every window;
median ms per step), with the SM clock sampled as bench.py does.  Then two deterministic runs of ``--check-steps`` steps
from the same state and seed are compared bit for bit.  Prints one JSON line.

    python tools/bench_deterministic.py [--steps 20] [--rounds 5] [--warmup 5] [--check-steps 3]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # before the first cuBLAS handle

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import neumesh_b200 as nb  # noqa: E402
from neumesh_b200 import _lib, synth  # noqa: E402

N_RAYS = 512
KW = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True, detailed_output=True, perturb=True)


def _card():
    """name, power limit and max SM clock of GPU 0 (read-only nvidia-smi query)."""
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--check-steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    grid = nb.MeshGrid(mesh, dev)

    def fresh():
        m = nb.NeuMesh(grid, **cfg.model_kwargs())
        m.load_state_dict(copy.deepcopy(sd))
        m = m.to(dev).train()
        return m, torch.optim.Adam(m.parameters(), lr=5e-4)

    model, opt = fresh()
    normals0 = grid.get_vertex_normal_torch().detach().clone()
    g = torch.Generator().manual_seed(1234)
    batches = []
    for i in range(16):
        o, d = synth.frame_rays(800, 800, view=i)
        sel = torch.randint(0, o.shape[0], (N_RAYS,), generator=g)
        batches.append(tuple(t.to(dev) for t in (o[sel], d[sel], torch.rand(N_RAYS, 3, generator=g),
                                                 (torch.rand(N_RAYS, generator=g) > 0.5).float())))

    def step(model, opt, i):
        o, d, tgt, msk = batches[i % len(batches)]
        opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, **KW)
        nab = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        loss = F.l1_loss(rgb, tgt) + 0.1 * F.mse_loss(nab, torch.ones_like(nab)) \
            + 0.1 * F.binary_cross_entropy(acc, msk) + 0.01 * F.mse_loss(model.indicator_vector, normals0)
        loss.backward()
        opt.step()

    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.wait_ready()
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        for i in range(args.warmup):
            step(model, opt, i)
    torch.cuda.synchronize()
    sampler.mark()
    ms = {False: [], True: []}
    launches = {}
    for r in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = _lib.launch_count()
            e0.record()
            for i in range(args.steps):
                step(model, opt, r * args.steps + i)
            e1.record()
            torch.cuda.synchronize()
            launches[det] = (_lib.launch_count() - l0) // args.steps
            ms[det].append(e0.elapsed_time(e1) / args.steps)
    clocks = sampler.stop()

    # bit identity of two deterministic runs from the same state
    torch.use_deterministic_algorithms(True)
    runs = []
    for _ in range(2):
        torch.manual_seed(7)
        m, o = fresh()
        for i in range(args.check_steps):
            step(m, o, i)
        torch.cuda.synchronize()
        runs.append({k: p.detach().clone() for k, p in m.named_parameters()})
    identical = all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])
    torch.use_deterministic_algorithms(False)

    props = torch.cuda.get_device_properties(dev)
    off, on = statistics.median(ms[False]), statistics.median(ms[True])
    print(json.dumps({
        "metric": "train_step_ms_deterministic_vs_default", "gpu": props.name,
        "card": _card(),
        "default_ms_per_step": off, "deterministic_ms_per_step": on, "extra_ms_per_step": on - off,
        "default_ms_rounds": ms[False], "deterministic_ms_rounds": ms[True],
        "library_launches_per_step": {"default": launches[False], "deterministic": launches[True]},
        "steps_per_round": args.steps, "rounds": args.rounds, "clocks": clocks,
        "deterministic_runs_bit_identical": identical, "check_steps": args.check_steps}), flush=True)
    if not identical:
        sys.exit(1)


if __name__ == "__main__":
    main()
