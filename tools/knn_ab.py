"""A/B check of the KNN kernels on a GPU: run once per variant (env NMB_KNN_LEGACY=1 / NMB_KNN_NO_DIR=1 / default),
each run dumps neighbour lists + mesh distances + a small render to ``<temp dir>/knn_ab/<tag>.pt``; ``compare`` then checks
that the variants agree (neighbour slots, ds and w bit for bit; the closed-form gradient to rounding).

    python tools/knn_ab.py dump <tag>
    python tools/knn_ab.py compare <tagA> <tagB>
"""
import os
import sys
import tempfile

import torch

OUT = os.path.join(tempfile.gettempdir(), "knn_ab")   # dumps of the variants, outside the source tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def dump(tag):
    import neumesh_b200 as nb
    from neumesh_b200 import synth
    from neumesh_b200.renderer import render_fused
    import helpers
    dev = torch.device("cuda:0")
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05")
    x, _ = helpers.sample_points(200000, seed=3)
    ind = sd["indicator_vector"].to(dev)
    ds, idx, w, grad = model.mesh_grid.grid.mesh_distance(x.to(dev), ind, 0.1, want_grad=True)
    o, d = synth.frame_rays(800, 800, view=0)
    sel = torch.arange(0, 640000, 9)[:60000]
    o, d = o[sel].to(dev), d[sel].to(dev)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True)
    with torch.no_grad():
        a = render_fused(o, d, model, chunk=60000, detailed_output=True, **kw)       # ray-ordered kernels + certificate
        b = render_fused(o[:1500], d[:1500], model, chunk=1500, detailed_output=False, **kw)   # per-point kernels
        c = render_fused(o, d, model, chunk=60000, detailed_output=False, **kw)      # live-sample lists
    torch.cuda.synchronize()
    out = {"ds": ds.cpu(), "idx": idx.cpu(), "w": w.cpu(), "grad": grad.cpu(), "near_far": a["near_far"].cpu(),
           "d_all": a["d_all"].cpu(), "sdf": a["implicit_surface"].cpu(), "rgb_full": a["rgb"].cpu(),
           "rgb_small": b["rgb"].cpu(), "depth_small": b["depth_volume"].cpu(), "rgb_live": c["rgb"].cpu(),
           "depth_live": c["depth_volume"].cpu(), "normals_live": c["normals_volume"].cpu()}
    os.makedirs(OUT, exist_ok=True)
    torch.save(out, os.path.join(OUT, f"{tag}.pt"))
    print(f"[{tag}] dumped; ds mean {ds.mean().item():.6f}")


def compare(ta, tb):
    a = torch.load(os.path.join(OUT, f"{ta}.pt"))
    b = torch.load(os.path.join(OUT, f"{tb}.pt"))
    ok = True
    for k in a:
        eq = torch.equal(a[k], b[k])
        err = (a[k].double() - b[k].double()).abs().max().item()
        print(f"{ta} vs {tb}: {k:14s} bit-identical {eq}  max-abs diff {err:.3e}")
        if k in ("ds", "idx", "w", "near_far", "d_all", "sdf") and not eq:
            ok = False
    print("AB", "OK" if ok else "MISMATCH")
    return 0 if ok else 1


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
