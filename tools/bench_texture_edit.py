"""Cost of a texture-edited frame (editing/texture_neumesh) against a plain frame, one JSON line.

Scene: main model on synth.icosphere_mesh(7) (V = 163 842, default config), two reference models on other icospheres,
two overlapping painted caps on the main mesh (about 30 % and 20 % of its vertices), main -> reference rotations, one
800 x 800 spiral frame, calc_normal + white background + bounded near/far (bench.py's RENDER_KW).  Timed with CUDA
events, median over --steps after --warmup:
  (a) plain fused render of the main model            (nmb_render)
  (b) fused edit render                               (nmb_render_edit)
  (c) the generic route (fused_render = False, rayschunk = 4096 as render.py passes): fused cascade, then the edit
      model's torch-op evaluation chunk by chunk
Also: the fraction of live samples each reference paints and the extra colour-MLP points (profile class "color").

    python tools/bench_texture_edit.py --steps 5 --warmup 2 --generic-steps 1
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import neumesh_b200 as nb  # noqa: E402
from neumesh_b200 import _lib, synth  # noqa: E402


def build_scene(dev):
    cfg = synth.ModelConfig()

    def model(level, seed):
        mesh = synth.icosphere_mesh(level, seed=seed)
        m = nb.NeuMesh(nb.MeshGrid(mesh, dev), **cfg.model_kwargs())
        m.load_state_dict(synth.make_state_dict(mesh, cfg, seed=seed + 1), strict=True)
        return mesh, m.to(dev).eval()

    mesh, main = model(7, 0)
    refs = [model(5, 10)[1], model(4, 20)[1]]
    v = torch.from_numpy(mesh.vertices).float()
    masks = torch.stack([v[:, 0] > 0.2, v[:, 2] > 0.3])     # caps of ~30 % and ~20 % of the vertices, overlapping
    g = torch.Generator().manual_seed(7)
    codes = torch.randn(v.shape[0], cfg.color_dim, generator=g)
    T = []
    for _ in range(2):
        q, _r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        if torch.det(q) < 0:
            q[:, 0] = -q[:, 0]
        t = torch.eye(4)
        t[:3, :3] = q.float()
        T.append(t.to(dev))
    edit = nb.TextureEditableNeuMesh(main, refs, masks.to(dev), codes.to(dev), T).to(dev).eval()
    return main, refs, masks, codes, T, edit


def time_render(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def colour_points(fn):
    fn()
    torch.cuda.synchronize()
    _lib.profile_collect()
    _lib.profile_enable(True)
    fn()
    prof = _lib.profile_collect()
    _lib.profile_enable(False)
    return prof["color"]["points"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=1, help="timed steps of the (slow) generic route (c)")
    ap.add_argument("--image", type=int, default=800)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_texture_edit needs a CUDA device")
    dev = torch.device("cuda:0")
    main_m, refs, masks, codes, T, edit = build_scene(dev)
    o, d = synth.frame_rays(args.image, args.image, view=0)
    o, d = o.to(dev), d.to(dev)
    kw = dict(bench.RENDER_KW, detailed_output=False)

    def render(model, **extra):
        with torch.no_grad():
            return nb.volume_render(o, d, model, **kw, **extra)

    def generic():
        edit.fused_render = False
        try:
            return render(edit, rayschunk=4096)
        finally:
            edit.fused_render = True

    clocks = bench.ClockSampler(0)
    clocks.start()
    clocks.wait_ready()
    render(main_m)
    render(edit)
    clocks.mark()
    ms_a = time_render(lambda: render(main_m), args.steps, args.warmup)
    ms_b = time_render(lambda: render(edit), args.steps, args.warmup)
    ms_c = time_render(generic, args.generic_steps, 1 if args.warmup else 0)
    clk = clocks.stop()
    # outputs of (b) against (c): the routes normalise the directions differently before the (rounding-sensitive)
    # sampling cascade, so a few rays move; report the share within the 1e-4 colour bar
    rgb_b, rgb_c = render(edit)[0], generic()[0]
    within = float(((rgb_b - rgb_c).abs().amax(-1) <= 1e-4).float().mean())
    # live colour points of the plain frame and the extra points each reference paints
    live = colour_points(lambda: render(main_m))
    extra = colour_points(lambda: render(edit)) - live
    per_ref = []
    for i in range(len(refs)):
        one = nb.TextureEditableNeuMesh(main_m, [refs[i]], masks[i:i + 1].to(dev), codes.to(dev), [T[i]]).eval()
        per_ref.append((colour_points(lambda: render(one)) - live) / max(live, 1))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power_limit = float(q.splitlines()[0])
    except Exception:
        power_limit = None
    print(json.dumps({
        "workload": f"texture_edit_{args.image}x{args.image}_icosphere_V163842_2refs",
        "plain_ms": round(ms_a, 2), "edit_ms": round(ms_b, 2), "generic_edit_ms": round(ms_c, 2),
        "edit_over_plain": round(ms_b / ms_a, 3), "generic_over_edit": round(ms_c / ms_b, 2),
        "painted_live_fraction": [round(f, 4) for f in per_ref], "live_colour_points": int(live),
        "extra_colour_points": int(extra), "painted_vertex_fraction": [round(float(m.float().mean()), 4) for m in masks],
        "fused_vs_generic_rays_within_1e-4": round(within, 4),
        "steps": args.steps, "generic_steps": args.generic_steps, "gpu": torch.cuda.get_device_name(0),
        "power_limit_w": power_limit, "clocks": clk}))


if __name__ == "__main__":
    main()
