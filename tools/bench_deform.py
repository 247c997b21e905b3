"""Cost of one geometry-editing frame (editing/render_geometry_editing.py:37-67, deform_model) on the device route
against the host route, one JSON line.

Scene: a NeuMesh model (default config) on synth.icosphere_mesh(7) (V = 163 842) and on the 2.6 M-vertex mesh of
bench.py's `--workload big` (synth.icosphere_mesh(9)), a wave displacement whose phase moves every frame, one
--image x --image spiral frame with bench.py's RENDER_KW (calc_normal, white background, bounded near/far).
Timed with CUDA events (each timed call ends in a device synchronise), median over --steps after --warmup:
  deform_render  deform_model(CUDA vertices) in place (nmb_grid_update, nmb_vertex_normals, nmb_indicator_rotate),
                 then the render, which re-packs the field (nmb_field_update) and rebuilds the shell certificate
  host_render    the host route: area-weighted normals of the deformed mesh on the CPU (what Open3D's
                 compute_vertex_normals gives the reference), deform_model(host mesh) = new MeshGrid (H2D copy,
                 nmb_grid_create) + indicator rotation, then the render (nmb_field_create + certificate + frame)
  render         the render alone, nothing changed since the previous one
and each update step on its own (grid_update, normals, rotate, field_update, shell).  Meshes not run are reported as
"not measured".

    python tools/bench_deform.py --steps 5 --warmup 2 --meshes icosphere,big
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import neumesh_b200 as nb  # noqa: E402
from neumesh_b200 import synth  # noqa: E402
from neumesh_b200.renderer import vertex_normals  # noqa: E402

MESHES = {"icosphere": 7, "big": 9}


def wave(v, phase):
    r = v.norm(dim=-1, keepdim=True)
    return v + 0.04 * torch.sin(8.0 * v[:, 0:1] + 6.0 * v[:, 1:2] + phase) * v / r


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def median_ms(make_fn, steps, warmup):
    """make_fn(i) -> the callable of step i (warm-up steps first, each with its own i)."""
    for i in range(warmup):
        timed(make_fn(i))
    return statistics.median(timed(make_fn(warmup + i)) for i in range(steps))


def run_mesh(level, dev, o, d, steps, warmup):
    cfg = synth.ModelConfig()
    t0 = time.time()
    mesh = synth.icosphere_mesh(level, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    print(f"level {level}: mesh + state dict on the host in {time.time() - t0:.1f} s", file=sys.stderr)
    kw = dict(bench.RENDER_KW, detailed_output=False)

    def new_model(m):
        model = nb.NeuMesh(nb.MeshGrid(m, dev), **cfg.model_kwargs())
        model.load_state_dict(sd, strict=True)
        return model.to(dev).eval()

    def render(model):
        with torch.no_grad():
            return nb.volume_render(o, d, model, **kw)

    model = new_model(mesh)
    base = model.mesh_grid.vertices.clone()
    tri = torch.from_numpy(mesh.triangles).to(dev)
    render(model)
    out = {"V": int(base.shape[0])}
    out["render_ms"] = median_ms(lambda i: (lambda: render(model)), steps, warmup)

    def device_frame(i):
        v = wave(base, 0.3 * i)
        return lambda: (nb.deform_model(v, model, dev), render(model))

    out["deform_render_ms"] = median_ms(device_frame, steps, warmup)

    # the update steps on their own (inputs prepared outside the timed region)
    mg = model.mesh_grid
    steps_ms = {k: [] for k in ("grid_update", "normals", "rotate", "field_update", "shell")}
    for i in range(warmup + steps):
        v = wave(base, 0.3 * i + 0.15)
        n_old = mg.vertex_normals
        t = {"grid_update": timed(lambda: mg.grid.update(v))}
        holder = {}
        t["normals"] = timed(lambda: holder.update(n=vertex_normals(mg.vertices, tri)))
        mg.vertex_normals = holder["n"]
        t["rotate"] = timed(lambda: holder.update(r=nb.indicator_rotate(n_old, holder["n"], model.indicator_vector)))
        model.indicator_vector = torch.nn.Parameter(holder["r"])
        t["field_update"] = timed(lambda: model.packed_field())
        t["shell"] = timed(lambda: model.shell_free_grid())
        if i >= warmup:
            for k, x in t.items():
                steps_ms[k].append(x)
    out["steps_ms"] = {k: round(statistics.median(x), 3) for k, x in steps_ms.items()}

    # the host route: a deformed host mesh each frame (its vertices prepared outside the timed region)
    host_model = new_model(mesh)
    render(host_model)
    host_v = [wave(base, 0.3 * i + 0.1).double().cpu().numpy() for i in range(warmup + steps)]

    def host_frame(i):
        def fn():
            m = synth.SynthMesh(host_v[i], mesh.triangles, None)
            # new MeshGrid (compute_vertex_normals on the CPU, H2D, nmb_grid_create) + rotation
            nb.deform_model(m, host_model, dev)
            render(host_model)                           # new field (nmb_field_create) + certificate + frame
        return fn

    out["host_render_ms"] = median_ms(host_frame, steps, warmup)
    out["host_over_device"] = round(out["host_render_ms"] / out["deform_render_ms"], 2)
    for k in ("render_ms", "deform_render_ms", "host_render_ms"):
        out[k] = round(out[k], 2)
    out["deform_overhead_ms"] = round(out["deform_render_ms"] - out["render_ms"], 2)
    del model, host_model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--image", type=int, default=800)
    ap.add_argument("--meshes", default="icosphere,big", help="comma-separated subset of %s" % sorted(MESHES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_deform needs a CUDA device")
    dev = torch.device("cuda:0")
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power_limit = float(q.splitlines()[0])
    except Exception:
        power_limit = None
    o, d = synth.frame_rays(args.image, args.image, view=0)
    o, d = o.to(dev), d.to(dev)
    wanted = [m for m in args.meshes.split(",") if m]
    results = {}
    for name in MESHES:
        results[name] = run_mesh(MESHES[name], dev, o, d, args.steps, args.warmup) if name in wanted else "not measured"
    print(json.dumps({"workload": f"deform_wave_{args.image}x{args.image}", "meshes": results, "steps": args.steps,
                      "warmup": args.warmup, "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit}))


if __name__ == "__main__":
    main()
