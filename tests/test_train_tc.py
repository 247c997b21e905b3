"""The 3xTF32 tensor-core engine of the training path: ``train_engine="tf32x3"`` (``nmb_tr_gemm_tc``,
``csrc/train_tc.cu``) for the fused training op and the NeuS teacher.

Error model of one product C = A.B on the engine.  Each operand is split as x = x_hi + x_lo + r with x_hi = tf32(x),
x_lo = tf32(x - x_hi), |r| <= 2^-11 |x - x_hi| <= 2^-22 |x|, and the engine sums a_lo b_hi + a_hi b_lo + a_hi b_hi.  Per
product that drops a_lo b_lo and the two r terms: at most 3 x 2^-22 (1 + 2^-11) |a b| < 2^-20 |a b|.  The sums are fp32
accumulations (the tensor core truncates inside a K step of 16; the steps are added by round-to-nearest FADDs), so the
bound of an element is the fp32 bound of ``test_gemm_edges_vs_float64`` (4 sqrt(K) u sum|a b|, u = 6e-8, + 1e-6) plus
2^-20 sum|a b|, plus one fp32 rounding (2^-23 relative) of each epilogue addition (bias, accumulate).

The field op, the patterns, the entry points, the whole step and the teacher are held to the bars the fp32 engine meets
in ``test_train_envelope`` (2 x the fp32 yardstick + the same floors; the fixed bars on rows A, B, E), the step also to
the unmodified reference's golden gradients (relative L2 <= 1e-3 per parameter).

CPU (``-m "not gpu"``): ``train_engine`` validation, unchanged ``state_dict`` keys, and ``CudaPrims`` routing.
GPU (``-m gpu``): everything else.
"""
from __future__ import annotations

import contextlib
import functools
import math

import pytest
import torch

import helpers
import neumesh_b200 as nb
import test_train_envelope as env
import test_train_ops as tops
from neumesh_b200 import _lib, synth, train_ops
from neumesh_b200.neus import NeuS

ENGINE = "tf32x3"
U = 6e-8


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def _neumesh_cpu(**kw):
    return nb.NeuMesh(env._FakeCudaGrid(), **synth.ModelConfig().model_kwargs(), **kw)


def test_train_engine_validation_cpu():
    m = _neumesh_cpu()
    assert m.train_engine == "fp32"
    m.train_engine = ENGINE
    assert m.train_engine == ENGINE
    assert _neumesh_cpu(train_engine=ENGINE).train_engine == ENGINE
    for bad in ("tf32", "FP32", None, "tcgen05"):
        with pytest.raises(ValueError):
            m.train_engine = bad
        with pytest.raises(ValueError):
            _neumesh_cpu(train_engine=bad)
    assert m.train_engine == ENGINE

    n = NeuS(**helpers.NEUS_KW)
    assert n.train_engine == n.implicit_surface.train_engine == n.radiance_net.train_engine == "fp32"
    n.train_engine = ENGINE
    assert n.train_engine == n.implicit_surface.train_engine == n.radiance_net.train_engine == ENGINE
    assert NeuS(**helpers.NEUS_KW, train_engine=ENGINE).radiance_net.train_engine == ENGINE
    for bad in ("bf16", None):
        with pytest.raises(ValueError):
            n.train_engine = bad
        with pytest.raises(ValueError):
            NeuS(**helpers.NEUS_KW, train_engine=bad)
    assert n.train_engine == ENGINE


def test_state_dict_keys_unchanged_cpu():
    """The engine is not state: the keys are those of the default model and checkpoints load with strict=True both
    ways."""
    a, b = _neumesh_cpu(), _neumesh_cpu(train_engine=ENGINE)
    assert list(a.state_dict()) == list(b.state_dict())
    b.load_state_dict(a.state_dict(), strict=True)
    a.load_state_dict(b.state_dict(), strict=True)
    n0, n1 = NeuS(**helpers.NEUS_KW), NeuS(**helpers.NEUS_KW, train_engine=ENGINE)
    n1.train_engine = ENGINE
    assert list(n0.state_dict()) == list(n1.state_dict())
    n1.load_state_dict(n0.state_dict(), strict=True)
    n0.load_state_dict(n1.state_dict(), strict=True)


class _FakeLib:
    """Records which GEMM symbol each call reaches."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append(name)
            return 0
        return call


@pytest.mark.parametrize("engine,symbol", [("fp32", "nmb_tr_gemm"), (ENGINE, "nmb_tr_gemm_tc"), (None, "nmb_tr_gemm")])
def test_cuda_prims_routes_gemm_cpu(monkeypatch, engine, symbol):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "sync_deterministic", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(_lib, "ptr", lambda t: None)
    monkeypatch.setattr(_lib, "stream_ptr", lambda d=None: None)
    P = train_ops.CudaPrims("cuda:0") if engine is None else train_ops.CudaPrims("cuda:0", engine)
    x = torch.zeros(4, 256)
    P.gemm(x, 256, True, x, 256, True, x, 256, 4, 4, 256)
    P.softplus_fwd(x, x, x, x)
    assert fake.calls == [symbol, "nmb_tr_softplus_fwd"]
    with pytest.raises(ValueError):
        train_ops.CudaPrims("cuda:0", "tf32")


# ------------------------------------------------------------------------------------------------------------------
# GPU: the GEMM against float64
# ------------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _tc_split_plan(M, N, K):
    """nmb_tr_gemm_tc's split-K plan (csrc/train_tc.cu), a function of (M, N, K) only -> (splits first chosen, k_chunk,
    splits launched)."""
    tiles = -(-M // 128) * -(-N // 128)
    if tiles < 264 and K >= 4096:
        s0 = min(-(-264 // tiles), -(-K // 1024))
    else:
        return 1, K, 1
    if s0 <= 1:
        return s0, K, 1
    kc = -(-(-(-K // s0)) // 16) * 16
    return s0, kc, -(-K // kc)


def _gemm_check(P, M, N, K, a_kc, b_kc, use_bias=False, epi=0, acc=False, seed=0):
    """One nmb_tr_gemm_tc call with odd strides and ldc = N + 3 against float64 under the stated error model ->
    worst error / bound."""
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    lda, ldb = (K if a_kc else M) + 3, (K if b_kc else N) + 5
    A = torch.randn(max(M if a_kc else K, 1) * lda, generator=g, device=dev)
    B = torch.randn(max(N if b_kc else K, 1) * ldb, generator=g, device=dev)
    Am = (A[:M * lda].view(M, lda)[:, :K] if a_kc else A[:K * lda].view(K, lda)[:, :M].t()).double()
    Bm = (B[:N * ldb].view(N, ldb)[:, :K].t() if b_kc else B[:K * ldb].view(K, ldb)[:, :N]).double()
    bias = torch.randn(N, generator=g, device=dev) if use_bias else None
    mask = torch.randn(M, N + 2, generator=g, device=dev) if epi == 2 else None
    C0 = torch.randn(M, N + 3, generator=g, device=dev)
    C = C0.clone()
    P.gemm(A, lda, a_kc, B, ldb, b_kc, C, N + 3, M, N, K, bias=bias, epilogue=epi, mask=mask,
           ldmask=N + 2 if epi == 2 else 0, accumulate=acc)
    assert torch.equal(C[:, N:], C0[:, N:]), "wrote outside the N columns"
    ref = Am @ Bm
    absprod = Am.abs() @ Bm.abs()
    epi_terms = torch.zeros_like(ref)
    if bias is not None:
        ref = ref + bias.double()
        epi_terms = epi_terms + bias.double().abs() + ref.abs()
    if epi == 1:
        ref = ref.clamp_min(0)
    if epi == 2:
        ref = torch.where(mask[:, :N] > 0, ref, torch.zeros_like(ref))
    if acc:
        ref = ref + C0[:, :N].double()
        epi_terms = epi_terms + C0[:, :N].double().abs() + ref.abs()
    bound = absprod * (4 * math.sqrt(max(K, 1)) * U + 2.0 ** -20) + 2.0 ** -23 * epi_terms + 1e-6
    err = (C[:, :N].double() - ref).abs()
    ratio = (err / bound).max().item() if err.numel() else 0.0
    assert (err <= bound).all(), ((M, N, K), a_kc, b_kc, use_bias, epi, acc, _tc_split_plan(M, N, K), ratio)
    return ratio


LAYOUTS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("a_kc,b_kc", LAYOUTS)
def test_gemm_tc_epilogues_vs_float64(a_kc, b_kc):
    """Every epilogue with and without bias, accumulate on and off, at a shape across tile edges in every direction."""
    P = train_ops.CudaPrims(_dev(), ENGINE)
    worst = 0.0
    for use_bias in (False, True):
        for epi in (0, 1, 2):
            for acc in (False, True):
                worst = max(worst, _gemm_check(P, 129, 257, 177, a_kc, b_kc, use_bias, epi, acc, seed=epi))
    print(f"nmb_tr_gemm_tc epilogues {a_kc, b_kc}: worst error / bound {worst:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("a_kc,b_kc", LAYOUTS)
def test_gemm_tc_k_and_tile_edges_vs_float64(a_kc, b_kc):
    """K in {0, 1, 7, 8, 9, 17, 177, 207, 256} and M, N across the 128 x 128 tile and 64-row warpgroup edges."""
    P = train_ops.CudaPrims(_dev(), ENGINE)
    worst = 0.0
    for K in (0, 1, 7, 8, 9, 17, 177, 207, 256):
        worst = max(worst, _gemm_check(P, 65, 129, K, a_kc, b_kc, use_bias=K % 2 == 1, seed=K))
    edges = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257)
    for M in edges:
        for N in edges:
            worst = max(worst, _gemm_check(P, M, N, 17, a_kc, b_kc, seed=M * 1000 + N))
    print(f"nmb_tr_gemm_tc K / tile edges {a_kc, b_kc}: worst error / bound {worst:.2e}")


def _split_edges(M, N):
    """K at the split-K switch (4096), where ceil(K / 1024) reaches the tile-count cap, where the aligned chunk first
    launches fewer splits than chosen, and the bench's K = 130 560."""
    tiles = -(-M // 128) * -(-N // 128)
    cap_k = (-(-264 // tiles) - 1) * 1024
    ks = [4095, 4096, 4097, cap_k, cap_k + 1, 130560]
    shrink = next(K for k in range(20000) for K in (4096 + 16 * k - 1, 4096 + 16 * k + 1)
                  if _tc_split_plan(M, N, K)[2] < _tc_split_plan(M, N, K)[0])
    return ks + [shrink]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(256, 256), (256, 17)])
def test_gemm_tc_split_k_edges_vs_float64(M, N):
    """The weight-gradient shapes (A = dZ [K, M], B = X [K, N], neither K-contiguous) around every switch of the split
    plan, overwriting and accumulating."""
    P = train_ops.CudaPrims(_dev(), ENGINE)
    worst = 0.0
    ks = _split_edges(M, N)
    plans = [_tc_split_plan(M, N, K) for K in ks]
    assert plans[0][2] == 1 and plans[1][2] > 1 and any(p[2] < p[0] for p in plans)
    for K in ks:
        for acc in (False, True):
            worst = max(worst, _gemm_check(P, M, N, K, False, False, acc=acc, seed=K))
    print(f"nmb_tr_gemm_tc split-K {M}x{N}: K {ks}, plans {plans}, worst error / bound {worst:.2e}")


@pytest.mark.gpu
def test_gemm_tc_k0_leaves_or_sets_c():
    """K = 0: C is the bias (or zero), or unchanged when accumulating; columns beyond N untouched."""
    dev = _dev()
    P = train_ops.CudaPrims(dev, ENGINE)
    one = torch.ones(1, device=dev)
    bias = torch.randn(7, device=dev)
    C0 = torch.randn(5, 9, device=dev)
    C = C0.clone()
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0, bias=bias)
    assert torch.equal(C[:, :7], bias.expand(5, 7)) and torch.equal(C[:, 7:], C0[:, 7:])
    C = C0.clone()
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0, accumulate=True)
    assert torch.equal(C, C0)
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0)
    assert (C[:, :7] == 0).all() and torch.equal(C[:, 7:], C0[:, 7:])


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True])
def test_gemm_tc_bit_identical_repeats(deterministic):
    """The same call twice gives the same bits, with torch's deterministic flag off and on (split-K and not)."""
    dev = _dev()
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(deterministic, warn_only=True)
    try:
        P = train_ops.CudaPrims(dev, ENGINE)
        g = torch.Generator(device=dev).manual_seed(7)
        for (M, N, K, a_kc, b_kc) in ((256, 207, 130560, False, False), (4099, 256, 177, True, True)):
            A = torch.randn((M if a_kc else K) * (K if a_kc else M), generator=g, device=dev)
            B = torch.randn((N if b_kc else K) * (K if b_kc else N), generator=g, device=dev)
            out = []
            for _ in range(2):
                C = torch.empty(M, N, device=dev)
                P.gemm(A, K if a_kc else M, a_kc, B, K if b_kc else N, b_kc, C, N, M, N, K)
                out.append(C)
            assert torch.equal(out[0], out[1]), (M, N, K)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the field op, the upstream patterns, the entry points with the engine
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _tc_model(row):
    cfg, mesh, sd = env._case(row)
    m = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    m.train_engine = ENGINE
    return m


def _tc_field_check(row, size_id):
    dev = _dev()
    cfg, mesh, sd = env._case(row)
    M = env._sizes()[size_id]
    model = _tc_model(row)
    x, v = env._off_relu_kinks(row, model, *env._points(M, mesh, seed=15), seed=15)
    up = env._upstream(M, seed=16)
    n0 = nb._lib.launch_count()
    got, idx, w = env._fused_run(model, x.to(dev), v.to(dev), up)
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 >= 10, "the field op did not run on the library's kernels"
    ref = env._reference_run(row, torch.float64, dev, x, v, idx, w, up)
    yard = env._reference_run(row, torch.float32, dev, x, v, idx, w, up)
    env._compare(f"gpu tf32x3 {row} M={M}", got, ref, yard, env.GPU_FLOOR_FWD, env.GPU_FLOOR_GRAD,
                 fixed=row in env.FIXED_BAR_ROWS, bands=cfg.multires_d)


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(env.MATRIX))
def test_tc_field_op_matrix_vs_float64(row):
    _tc_field_check(row, env.MID_SIZE)


@pytest.mark.gpu
@pytest.mark.parametrize("size_id", [s for s in env.SIZE_IDS if s != env.MID_SIZE])
@pytest.mark.parametrize("row", ["A", "F"])
def test_tc_field_op_batch_sizes_vs_float64(row, size_id):
    _tc_field_check(row, size_id)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(env.PATTERNS))
def test_tc_upstream_patterns_vs_float64(name):
    env._pattern_check(name, train_ops.CudaPrims(_dev(), ENGINE), _dev(), 3 * 32 * 132 + 5, env.GPU_FLOOR_FWD,
                       env.GPU_FLOOR_GRAD)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", env.ENTRIES)
def test_tc_grad_mode_entry_points_vs_float64(entry):
    dev = _dev()
    cfg, mesh, sd = env._case("A")
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    model.train_engine = ENGINE
    ref_model = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    ref_model.load_state_dict(sd)
    res = env._api_patterns(entry, model, ref_model.to(dev), mesh, dev)
    if res is not None:
        env._compare(f"gpu tf32x3 entry {entry}", *res, env.GPU_FLOOR_FWD, env.GPU_FLOOR_GRAD, fixed=True)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the whole training step
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", env.STEP_ROWS)
def test_tc_train_step_vs_float64(row, golden_dir):
    dev = _dev()
    model = _tc_model(row)
    o, d, z = env._step_rays(golden_dir)
    if model.fused_supported():
        with torch.no_grad():
            _, _, ex = nb.volume_render(o.to(dev), d.to(dev), model, rayschunk=4096, **helpers.TRAIN_KW)
        z = ex["d_all"].cpu()
    got = env._step(model, o.to(dev), d.to(dev), z.to(dev))
    ref, yard = env._step_references(row, o, d, z)
    assert set(got) == set(ref)
    env._compare(f"gpu tf32x3 step {row}", got, ref, yard, env.STEP_FLOOR_FWD, env.STEP_FLOOR_GRAD)


@pytest.mark.gpu
def test_tc_train_step_vs_reference_golden(golden_dir):
    """The step at the reference's teacher-forced sample depths against the unmodified reference's gradients."""
    dev = _dev()
    g, cfg, mesh, sd = tops._load(golden_dir)
    o, d = torch.from_numpy(g["rays_o"]).to(dev), torch.from_numpy(g["rays_d"]).to(dev)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    model.train_engine = ENGINE
    rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, z_samples=torch.from_numpy(g["d_all"]).to(dev),
                                      **helpers.TRAIN_KW)
    loss = helpers.train_loss(rgb, depth, ex)
    loss.backward()
    worst = tops._check(g, loss.item(), dict(model.named_parameters()), rtol=1e-3, l2tol=1e-3)
    print(f"tf32x3 training step vs reference golden gradients: worst relative L2 {worst:.2e}")


# ------------------------------------------------------------------------------------------------------------------
# GPU: the NeuS teacher
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 4099])
@pytest.mark.parametrize("case", list(env.NEUS_CASES))
def test_tc_neus_teacher_vs_float64(case, M, monkeypatch):
    dev = _dev()
    m = env._neus(case)
    x, v = env._neus_points(M, seed=61)
    ref = env._neus_eval(m.double(), x.double(), v.double())
    yard = env._neus_eval(m.float(), x, v)
    md = m.to(dev)
    md.train_engine = ENGINE
    calls = []
    gemm = train_ops.CudaPrims.gemm

    def counted(self, *a, **k):
        calls.append(self.gemm_symbol)
        return gemm(self, *a, **k)
    monkeypatch.setattr(train_ops.CudaPrims, "gemm", counted)
    with torch.no_grad():
        got = env._neus_eval(md, x.to(dev), v.to(dev))
    torch.cuda.synchronize()
    assert calls and set(calls) == {"nmb_tr_gemm_tc"}, calls
    assert len(calls) == md.implicit_surface.D + 1 + md.radiance_net.D + 1
    got = {k: t.reshape(ref[k].shape) for k, t in got.items()}
    bad = []
    for k in ref:
        e, y = env._rel(got[k], ref[k], 1e-3), env._rel(yard[k], ref[k], 1e-3)
        print(f"[neus tf32x3 {case} M={M}] {k} {e:.1e}/{y:.1e}")
        if not e <= 2 * y + 1e-5:
            bad.append((k, e, y))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------
# GPU: reproducible training
# ------------------------------------------------------------------------------------------------------------------
def _adam_run(steps=5):
    dev = _dev()
    torch.manual_seed(1234)
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(5, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = nb.NeuMesh(nb.MeshGrid(mesh, dev), **cfg.model_kwargs(), train_engine=ENGINE)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    g = torch.Generator().manual_seed(1234)
    kw = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True, detailed_output=True, perturb=True)
    for i in range(steps):
        o, d = synth.frame_rays(200, 200, view=i)
        sel = torch.randint(0, o.shape[0], (512,), generator=g)
        tgt = torch.rand(512, 3, generator=g).to(dev)
        opt.zero_grad(set_to_none=True)
        rgb, depth, ex = nb.volume_render(o[sel].to(dev), d[sel].to(dev), model, rayschunk=4096, **kw)
        nab = ex["implicit_nablas"].norm(dim=-1)
        loss = (rgb - tgt).abs().mean() + 0.1 * ((nab - 1.0) ** 2).mean()
        loss.backward()
        opt.step()
    return {k: p.detach().clone() for k, p in model.named_parameters()}


@pytest.mark.gpu
def test_tc_adam_steps_bit_identical_deterministic():
    """Under torch.use_deterministic_algorithms(True) two runs of five Adam steps with the engine give the same bits."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a, b = _adam_run(), _adam_run()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
