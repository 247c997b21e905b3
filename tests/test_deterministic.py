"""``torch.use_deterministic_algorithms(True)`` on the fused training op and the vertex normals.

Under torch's flag the reducing kernels of ``csrc/train.cu`` and ``nmb_vertex_normals`` switch to summation orders that
are a function of their inputs alone (sorted segmented scatter, fixed row partitions, an SM-independent split-K plan):
repeated calls are bit-identical, and their error against float64 stays inside the bars the atomic path meets.  With the
flag off nothing changes: same launches, same kernels."""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import test_train_envelope as env
import test_train_ops as tops
from neumesh_b200 import _lib, synth, train_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPEATS = 5


@pytest.fixture
def deterministic():
    """torch's flag on (warn_only: the float64 references below use ops torch has no deterministic kernel for), then
    restored."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _dev():
    return torch.device("cuda:0")


def _rows(t, M, dev):
    """The first M rows of t (M + 1 rows) on dev: a non-null device pointer also at M = 0."""
    return t.to(dev)[:M]


def _repeat_equal(fn):
    """fn() -> tuple of tensors, run REPEATS times on identical inputs; every run must match the first bit for bit."""
    first = [t.clone() for t in fn()]
    for _ in range(REPEATS - 1):
        for a, b in zip(first, fn()):
            assert torch.equal(a, b)
    return first


# ---- host ---------------------------------------------------------------------------------------------------------
class _RecordingLib:
    """Stands in for the library's nmb_tr_* entry points; records the real library's mode at every call."""

    def __init__(self):
        self.modes = []

    def __getattr__(self, name):
        def call(*args):
            self.modes.append((name, int(_lib.lib().nmb_deterministic())))
            return 0
        return call


def test_cuda_prims_follow_torch_flag_cpu(monkeypatch):
    """Every reducing CudaPrims call sets the library mode from torch's flag, also when the flag changes between calls."""
    import contextlib
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(_lib, "ptr", lambda t: None)
    monkeypatch.setattr(_lib, "stream_ptr", lambda d=None: None)
    monkeypatch.setattr(train_ops.CudaPrims, "_inputs", lambda self, spec, t: train_ops.TrInputs())
    P = train_ops.CudaPrims("cuda:0")
    P.L = rec = _RecordingLib()
    x = torch.zeros(4, 256)
    calls = [lambda: P.gemm(x, 256, True, x, 256, True, x, 256, 4, 4, 256),
             lambda: P.colsum(x, x[0]),
             lambda: P.color_out_bwd(x, x, x, x, x, x, x),
             lambda: P.geo_out_bwd(x, x, None, x, x, x, x, x, x, x, x, x, x),
             lambda: P.input_bwd(None, {}, x, x, x, x, x, x, x, x)]
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        want = []
        for i, flag in enumerate([True, False, True, True, False] * 2):
            if flag and i % 2:
                torch.use_deterministic_algorithms(True, warn_only=True)   # warn_only counts as on
            else:
                torch.use_deterministic_algorithms(flag)
            calls[i % len(calls)]()
            want.append(int(flag))
        assert [m for _, m in rec.modes] == want, rec.modes
        assert [n for n, _ in rec.modes][:5] == ["nmb_tr_gemm", "nmb_tr_colsum", "nmb_tr_color_out_bwd",
                                                 "nmb_tr_geo_out_bwd", "nmb_tr_input_bwd"]
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
        _lib.sync_deterministic()
    assert _lib.lib().nmb_deterministic() == int(prev)


def test_mode_symbols_cpu():
    L = _lib.lib()
    prev = L.nmb_deterministic()
    try:
        L.nmb_set_deterministic(7)
        assert L.nmb_deterministic() == 1
        L.nmb_set_deterministic(0)
        assert L.nmb_deterministic() == 0
    finally:
        L.nmb_set_deterministic(prev)


# ---- per kernel, flag on --------------------------------------------------------------------------------------------
def _sum_bound(M, absum):
    """fp32 summation bound of the fixed-partition reductions: the rows one thread adds, the 8-way and the block-order
    levels (as test_colsum_many_rows_vs_float64)."""
    terms = -(-M // (8 * 512)) + 8 + 512
    return terms * 6e-8 * absum + 1e-30


ROW_COUNTS = [1, 7, 4097, 512 * 8 * 3 + 5, 70001]   # M = 0: test_zero_rows_deterministic


@pytest.mark.gpu
def test_colsum_deterministic(deterministic):
    env.test_colsum_many_rows_vs_float64()
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    g = torch.Generator().manual_seed(61)
    for M in ROW_COUNTS:
        for N in (1, 33, 256):
            X = _rows(torch.randn(M + 1, N, generator=g) + 0.5, M, dev)
            base = torch.full((N,), 0.25, device=dev)

            def run():
                out = base.clone()
                P.colsum(X, out)
                return (out,)
            (out,) = _repeat_equal(run)
            ref = X.double().sum(0) + 0.25
            assert ((out.double() - ref).abs() <= _sum_bound(M, X.double().abs().sum(0))).all(), (M, N)


@pytest.mark.gpu
def test_color_out_bwd_deterministic(deterministic):
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    g = torch.Generator().manual_seed(62)
    for M in ROW_COUNTS:
        b_rgb, rgb = _rows(torch.randn(M + 1, 3, generator=g), M, dev), _rows(torch.rand(M + 1, 3, generator=g), M, dev)
        c, W = _rows(torch.randn(M + 1, 256, generator=g).relu(), M, dev), torch.randn(3, 256, generator=g).to(dev)

        def run():
            bz = _rows(torch.empty(M + 1, 256), M, dev)
            dw, db = torch.zeros(3, 256, device=dev), torch.zeros(3, device=dev)
            P.color_out_bwd(b_rgb, rgb, c, W, bz, dw, db)
            return bz, dw, db
        bz, dw, db = _repeat_equal(run)
        bo = b_rgb.double() * rgb.double() * (1 - rgb.double())
        assert ((dw.double() - bo.t() @ c.double()).abs() <= _sum_bound(M, bo.abs().t() @ c.double().abs())).all(), M
        assert ((db.double() - bo.sum(0)).abs() <= _sum_bound(M, bo.abs().sum(0))).all(), M
        if M:
            assert torch.allclose(bz.double(), (bo @ W.double()) * (c > 0), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_geo_out_bwd_deterministic(deterministic):
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    g = torch.Generator().manual_seed(63)
    for M in ROW_COUNTS:
        b_sdf, b_nab, G, gg, h, t = (_rows(torch.randn(M + 1, *s, generator=g), M, dev)
                                     for s in ((), (3,), (3,), (), (256,), (256,)))
        w = torch.randn(1, 256, generator=g).to(dev)

        def run():
            bh, bt, bG = (_rows(torch.empty(M + 1, k), M, dev) for k in (256, 256, 3))
            dw, db = torch.zeros(1, 256, device=dev), torch.zeros(1, device=dev)
            P.geo_out_bwd(b_sdf, b_nab, None, G, gg, h, t, w, bh, bt, bG, dw, db)
            return dw, db
        dw, db = _repeat_equal(run)
        bs, bg = b_sdf.double(), (b_nab.double() * G.double()).sum(-1)
        ref = bs @ h.double() + bg @ t.double()
        absum = bs.abs() @ h.double().abs() + bg.abs() @ t.double().abs()
        assert ((dw[0].double() - ref).abs() <= _sum_bound(M, absum) + 1e-6 * absum).all(), M
        assert (db.double() - bs.sum()).abs().item() <= _sum_bound(M, bs.abs().sum()).item(), M


@pytest.mark.gpu
def test_gemm_split_k_deterministic(deterministic):
    env.test_gemm_edges_vs_float64()
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    g = torch.Generator().manual_seed(64)
    # split-K plans of the weight gradients (the plan is the one for 132 SMs on any device)
    for (M, N, K) in [(256, 256, 4097), (256, 17, 4096 + 16 * 7 + 1), (256, 256, 130560), (1, 256, 5000), (1, 1, 4097)]:
        A, B = torch.randn(K, M, generator=g).to(dev), torch.randn(K, N, generator=g).to(dev)
        assert env._split_plan(M, N, K, 132)[2] > 1

        def run():
            C = torch.zeros(M, N, device=dev)
            P.gemm(A, M, False, B, N, False, C, N, M, N, K)
            return (C,)
        _repeat_equal(run)


def _scatter_case(F, M, V, seed):
    """Inputs of nmb_tr_prep / nmb_tr_input_bwd with codes of width F; half of the points share 8 neighbours.  Per-point
    tensors have M + 1 rows (see _on)."""
    g = torch.Generator().manual_seed(seed)
    spec = train_ops.FieldSpec(F, F, 6, 2, 2, 4, True, 3, 4)
    idx = torch.randint(0, V, (M + 1, 8), generator=g)
    idx[: M // 2] = torch.randperm(V, generator=g)[:8]
    w = torch.rand(M + 1, 8, generator=g) + 0.05
    t = dict(xyz=torch.randn(M + 1, 3, generator=g), dirs=torch.randn(M + 1, 3, generator=g), idx=idx,
             w=w / w.sum(-1, True),
             vertices=torch.randn(V, 3, generator=g), indicator_vector=torch.randn(V, 3, generator=g),
             geometry_features=torch.randn(V, F, generator=g), color_features=torch.randn(V, F, generator=g))
    up = {k: torch.randn(M + 1, n, generator=g) for k, n in (("bXg", spec.Kg), ("bT0", spec.chd), ("bXc", spec.Kc), ("b_G", 3))}
    return spec, t, up


def _on(d, dev, M):
    """_scatter_case's tensors on dev, the per-point ones cut to M rows."""
    return {k: _rows(v, M, dev) if k not in ("vertices", "indicator_vector", "geometry_features", "color_features")
            else v.to(dev) for k, v in d.items()}


def _input_bwd(P, spec, t, up, w1, M):
    V = t["vertices"].shape[0]
    S = _on(t, P.dev, M)
    S["w1"] = w1
    for k, shape in (("ds", ()), ("G", (3,)), ("Xg", (spec.Kg,)), ("T0", (spec.chd,)), ("Xc", (spec.Kc,))):
        S[k] = _rows(P.empty(M + 1, *shape), M, P.dev)
    P.prep(spec, S)
    out = P.zeros(V, spec.Fg), P.zeros(V, spec.Fc), P.zeros(V, 3), P.zeros(1)
    u = _on(up, P.dev, M)
    P.input_bwd(spec, S, u["bXg"], u["bT0"], u["bXc"], u["b_G"], *out)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("F", [32, 256])
def test_input_bwd_deterministic(deterministic, F):
    """Repeated calls bit-identical; against the same kernels in float64 (torch primitives) within twice the default
    (atomic) path's error plus a floor (the indicator-weight gradient cancels: its terms are ~30x the sum)."""
    from train_prims_torch import TorchPrims
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    for M in (1, 7, 3001):
        spec, t, up = _scatter_case(F, M, 97, seed=65 + F + M)
        got = _repeat_equal(lambda: _input_bwd(P, spec, t, up, 0.1, M))
        torch.use_deterministic_algorithms(False)
        yard = _input_bwd(P, spec, t, up, 0.1, M)
        torch.use_deterministic_algorithms(True, warn_only=True)
        R = TorchPrims(dev, torch.float64)
        ref = _input_bwd(R, spec, {k: v.double() if v.is_floating_point() else v for k, v in t.items()},
                         {k: v.double() for k, v in up.items()}, 0.1, M)
        for a, y, b in zip(got, yard, ref):
            bound = 2 * (y.double() - b).abs() + 1e-5 * b.abs().max()
            assert ((a.double() - b).abs() <= bound).all(), (F, M, ((a.double() - b).abs() - bound).max().item())


@pytest.mark.gpu
def test_zero_rows_deterministic(deterministic):
    """M = 0 through the C ABI (torch gives empty tensors a null pointer): every reducing call returns 0 and leaves its
    accumulated outputs as they were."""
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    L, s, p = _lib.lib(), _lib.stream_ptr(dev), _lib.ptr
    one = torch.ones(1, 256, device=dev)
    acc = torch.full((3, 256), 0.5, device=dev)
    before = acc.clone()
    for rc in (L.nmb_tr_colsum(p(one), 256, 0, 256, p(acc), s),
               L.nmb_tr_color_out_bwd(p(one), p(one), p(one), p(one), 0, 256, p(one), p(acc), p(acc), s),
               L.nmb_tr_geo_out_bwd(p(one), p(one), None, 0, p(one), p(one), p(one), p(one), p(one), 0, 256, p(one),
                                    p(one), p(one), p(acc), p(acc), s),
               L.nmb_tr_gemm(p(one), 256, 0, p(one), 256, 0, p(acc), 256, 0, 256, 5000, None, 0, None, 0, 1, s)):
        assert rc == 0
    spec, t, up = _scatter_case(32, 1, 11, seed=73)
    S = _on(t, dev, 1)
    S["w1"] = 0.1
    for k, n in (("ds", 1), ("G", 3), ("Xg", spec.Kg), ("T0", spec.chd), ("Xc", spec.Kc)):
        S[k] = P.empty(1, n)
    ins = P._inputs(spec, S)
    ins.M = 0
    u = _on(up, dev, 1)
    outs = [torch.full((11, n), 0.5, device=dev) for n in (32, 32, 3)] + [torch.full((1,), 0.5, device=dev)]
    assert L.nmb_tr_input_bwd(ctypes.byref(ins), p(u["bXg"]), spec.Kg, p(u["bT0"]), spec.chd, p(u["bXc"]), spec.Kc,
                              p(u["b_G"]), *[p(o) for o in outs], s) == 0
    torch.cuda.synchronize()
    assert torch.equal(acc, before) and all((o == 0.5).all() for o in outs)


@pytest.mark.gpu
def test_input_bwd_cluster_deterministic(deterministic):
    """The 1e5-point cluster on 8 shared rows (runs of 1e5 entries) within the atomic path's bound, and bit-identical."""
    env.test_atomic_scatter_cluster_vs_float64()
    dev = _dev()
    model = env._gpu_model("A")
    cfg, mesh, sd = env._case("A")
    x, v = env._points(20000, mesh, seed=66)
    up = env._upstream(20000, seed=67)
    first = None
    for _ in range(REPEATS):
        got, _, _ = env._fused_run(model, x.to(dev), v.to(dev), up)
        got = {k: t.detach().clone() for k, t in got.items()}
        if first is None:
            first = got
        assert all(torch.equal(first[k], got[k]) for k in first)


@pytest.mark.gpu
def test_vertex_normals_deterministic(deterministic):
    from neumesh_b200.renderer import vertex_normals
    dev = _dev()
    for mesh in (synth.icosphere_mesh(5, seed=0), synth.icosphere_mesh(7, seed=0)):
        vt = torch.from_numpy(mesh.vertices).float().to(dev)
        tri = torch.from_numpy(mesh.triangles).to(dev)
        (n,) = _repeat_equal(lambda: (vertex_normals(vt, tri),))
        assert (n.cpu().double() - torch.from_numpy(mesh.vertex_normals)).abs().max() < 2e-4


# ---- the whole op ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", list(env.MATRIX))
def test_fused_field_fn_bit_identical(deterministic, row):
    dev = _dev()
    cfg, mesh, sd = env._case(row)
    model = env._gpu_model(row)
    M = env._sizes()[env.MID_SIZE]
    x, v = env._points(M, mesh, seed=68)
    up = env._upstream(M, seed=69)
    a, _, _ = env._fused_run(model, x.to(dev), v.to(dev), up)
    a = {k: t.detach().clone() for k, t in a.items()}
    b, _, _ = env._fused_run(model, x.to(dev), v.to(dev), up)
    for k in a:
        assert torch.equal(a[k], b[k]), (row, k)


@pytest.mark.gpu
def test_train_step_golden_deterministic(deterministic, golden_dir):
    tops.test_train_step_fused_cuda_vs_reference_golden(golden_dir)


# ---- default path unchanged ------------------------------------------------------------------------------------------
class _CountingPrims(train_ops.CudaPrims):
    """The launches the default path makes: one per kernel call on M > 0 rows, two for a split-K GEMM."""

    def __init__(self, dev):
        super().__init__(dev)
        self.expected = 0
        self.sms = torch.cuda.get_device_properties(self.dev).multi_processor_count

    def gemm(self, A, lda, a_kc, B, ldb, b_kc, Cm, ldc, M, N, K, bias=None, epilogue=0, mask=None, ldmask=0,
             accumulate=False):
        if M > 0 and N > 0:
            split = bias is None and epilogue == 0 and env._split_plan(M, N, K, self.sms)[2] > 1
            self.expected += 2 if split else 1
        super().gemm(A, lda, a_kc, B, ldb, b_kc, Cm, ldc, M, N, K, bias, epilogue, mask, ldmask, accumulate)


for _name in ("color_out_bwd", "colsum", "geo_out_bwd", "softplus_bwd", "input_bwd"):
    def _counted(self, *a, _f=getattr(train_ops.CudaPrims, _name)):
        self.expected += 1
        return _f(self, *a)
    setattr(_CountingPrims, _name, _counted)


@pytest.mark.gpu
def test_default_backward_launch_count():
    assert not torch.are_deterministic_algorithms_enabled()
    dev = _dev()
    M = 4097
    spec, t, _ = _scatter_case(32, M, 2000, seed=70)
    t = _on(t, dev, M)
    t["w1"] = 0.1
    P = _CountingPrims(dev)
    g = torch.Generator().manual_seed(71)
    geo = [(torch.randn(256, spec.Kg if l == 0 else 256, generator=g).to(dev) * 0.05,
            torch.randn(256, generator=g).to(dev) * 0.05) for l in range(spec.NLg)]
    col = [(torch.randn(256, spec.Kc if l == 0 else 256, generator=g).to(dev) * 0.05,
            torch.randn(256, generator=g).to(dev) * 0.05) for l in range(spec.NLc)]
    geo_out = (torch.randn(1, 256, generator=g).to(dev) * 0.05, torch.zeros(1, device=dev))
    col_out = (torch.randn(3, 256, generator=g).to(dev) * 0.05, torch.zeros(3, device=dev))
    _, _, _, S = train_ops.field_forward(P, spec, t, geo, geo_out, col, col_out)
    up = [u.to(dev) for u in env._upstream(M, seed=72)]
    P.expected = 0
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    train_ops.field_backward(P, spec, S, geo, geo_out, col, col_out, up[0].reshape(-1), up[1], up[2])
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == P.expected > 20


# ---- end to end, across processes ----------------------------------------------------------------------------------
_E2E = textwrap.dedent('''
    import os, sys
    import numpy as np
    import torch
    import torch.nn.functional as F
    sys.path.insert(0, sys.argv[2])
    torch.use_deterministic_algorithms(True)
    import neumesh_b200 as nb
    from neumesh_b200 import synth
    from neumesh_b200.deform import deform_model
    dev = torch.device("cuda:0")
    torch.manual_seed(1234)
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(7, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = nb.NeuMesh(nb.MeshGrid(mesh, dev), **cfg.model_kwargs())
    model.load_state_dict(sd)
    model = model.to(dev).train()
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    normals0 = model.mesh_grid.get_vertex_normal_torch().detach().clone()
    g = torch.Generator().manual_seed(1234)
    kw = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True, detailed_output=True, perturb=True)
    for i in range(3):
        o, d = synth.frame_rays(800, 800, view=i)
        sel = torch.randint(0, o.shape[0], (512,), generator=g)
        tgt, msk = torch.rand(512, 3, generator=g).to(dev), (torch.rand(512, generator=g) > 0.5).float().to(dev)
        opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o[sel].to(dev), d[sel].to(dev), model, rayschunk=4096, **kw)
        nab = ex["implicit_nablas"].norm(dim=-1)
        acc = ex["mask_volume"].clamp(1e-3, 1 - 1e-3)
        loss = F.l1_loss(rgb, tgt) + 0.1 * F.mse_loss(nab, torch.ones_like(nab)) \\
            + 0.1 * F.binary_cross_entropy(acc, msk) + 0.01 * F.mse_loss(model.indicator_vector, normals0)
        loss.backward()
        opt.step()
    out = {k: p.detach().cpu().numpy() for k, p in model.named_parameters()}
    v = torch.from_numpy(mesh.vertices).float().to(dev)
    moved = v * (1.0 + 0.05 * torch.sin(4.0 * v[:, :1]))
    deform_model(moved, model, dev)
    out["deformed_indicator_vector"] = model.indicator_vector.detach().cpu().numpy()
    np.savez(sys.argv[1], **out)
''')


@pytest.mark.gpu
def test_training_steps_bit_identical_across_processes(tmp_path):
    """Two fresh processes under torch.use_deterministic_algorithms(True): 3 training steps of the bench workload
    (V = 163 842, 512 rays, perturb=True, Adam) and one deform_model give byte-identical parameters."""
    envv = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    files = []
    for i in range(2):
        f = tmp_path / f"run{i}.npz"
        r = subprocess.run([sys.executable, "-c", _E2E, str(f), ROOT], env=envv, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr[-4000:]
        files.append(np.load(f))
    a, b = files
    assert set(a.files) == set(b.files) and "geometry_features" in a.files
    for k in a.files:
        assert a[k].tobytes() == b[k].tobytes(), k
