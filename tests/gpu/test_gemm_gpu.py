"""GPU tier: the wgmma GEMM against an fp32 reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(128, 256, 64), (256, 512, 128), (384, 768, 320), (1000, 1000, 264),
                                   (2048, 6144, 4096), (4096, 4096, 14336)])
def test_gemm_nt_matches_fp32(shape):
    from deepspeed_b200.ops.kernels import gemm_sm100
    M, N, K = shape
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    c = gemm_sm100.matmul_nt(a, b)
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    err = (c.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err < 1e-2 * scale + 1e-2, (err, scale)
    lib = torch.matmul(a, b.t())
    assert (c.float() - lib.float()).abs().max().item() < 2e-2 * scale + 1e-2


def test_gemm_strided_views_and_fewer_sms():
    from deepspeed_b200.ops.kernels import gemm_sm100
    torch.manual_seed(1)
    big_a = torch.randn(512, 1024, device="cuda", dtype=torch.bfloat16)
    big_b = torch.randn(1024, 1024, device="cuda", dtype=torch.bfloat16)
    a, b = big_a[:, 128:640], big_b[:, 256:768]  # row stride 1024, K = 512
    assert gemm_sm100.supports(a, b)
    c = gemm_sm100.matmul_nt(a, b, sms=7)
    ref = a.float() @ b.float().t()
    assert (c.float() - ref).abs().max().item() < 1e-2 * ref.abs().max().item() + 1e-2


@pytest.mark.parametrize("shape", [(256, 256, 64), (128, 256, 64), (512, 512, 128), (384, 768, 320), (1000, 1000, 264),
                                   (2048, 6144, 4096), (4096, 4096, 14336), (8192, 28672, 4096)])
def test_gemm_2cta_matches_fp32(shape):
    """General-entry kernel, including M/N edges that leave a tile partly or entirely outside the matrix."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    M, N, K = shape
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    c = gemm_sm100.matmul_nt_2cta(a, b)
    torch.cuda.synchronize()
    lib = torch.matmul(a, b.t())
    scale = lib.float().abs().max().item()
    assert (c.float() - lib.float()).abs().max().item() < 2e-2 * scale + 1e-2
    # repeated launches (barrier phases, registers double buffering across many tiles) stay correct
    for _ in range(3):
        c2 = gemm_sm100.matmul_nt_2cta(a, b)
    assert torch.equal(c, c2)


@pytest.mark.parametrize("shape", [(256, 256, 64), (512, 384, 192), (1000, 520, 264), (8192, 4096, 6144), (4096, 14336, 8192)])
def test_gemm_2cta_nn_tn_match_cublas(shape):
    """MN-major operands: NN (dX = dY W) and TN (dW = dY^T X), incl. strided views and writes into a larger buffer."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    M, N, K = shape
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b_kn = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    c = gemm_sm100.matmul_nn(a, b_kn)
    ref = torch.mm(a, b_kn)
    scale = ref.float().abs().max().item()
    assert (c.float() - ref.float()).abs().max().item() < 2e-2 * scale + 1e-2
    a_km = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    big = torch.zeros(M + 8, N + 16, device="cuda", dtype=torch.bfloat16)
    out = big[:M, 8:8 + N] if N % 8 == 0 else None
    c2 = gemm_sm100.matmul_tn(a_km, b_kn, out=out)
    ref2 = torch.mm(a_km.t(), b_kn)
    scale2 = ref2.float().abs().max().item()
    assert (c2.float() - ref2.float()).abs().max().item() < 2e-2 * scale2 + 1e-2
    if out is not None:
        assert float(big[M:].abs().max()) == 0.0 and float(big[:, :8].abs().max()) == 0.0


def test_flat_linear_backward_uses_native_gemm_and_matches_autograd():
    from deepspeed_b200.ops import gemm
    from deepspeed_b200.ops.linear import flat_linear
    torch.manual_seed(0)
    x = torch.randn(4, 512, 1024, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    w = torch.randn(2048, 1024, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    y = flat_linear(x, w)
    g = torch.randn_like(y)
    y.backward(g)
    xr, wr = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
    torch.nn.functional.linear(xr, wr).backward(g)
    for got, ref in ((x.grad, xr.grad), (w.grad, wr.grad)):
        s = ref.float().abs().max().item()
        assert (got.float() - ref.float()).abs().max().item() < 2e-2 * s + 1e-2
    assert any(k.split(":")[0] in ("nn", "tn") for k in gemm.tuning_table())


@pytest.mark.parametrize("counts", [[300, 0, 17, 128, 1, 513], [0, 0, 5, 0], [256, 256]])
@pytest.mark.parametrize("N,K", [(512, 256), (328, 192)])
def test_grouped_gemm_matches_per_expert_loop(counts, N, K):
    """Device-driven grouped wgmma GEMM (MoE): ragged expert extents incl. empty experts, N not a tile multiple."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    torch.manual_seed(0)
    E, rows = len(counts), sum(counts)
    x = (torch.randn(rows, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(E, N, K, device="cuda") * 0.1).bfloat16()
    off = torch.tensor([0] + list(torch.tensor(counts).cumsum(0)), dtype=torch.int32, device="cuda")
    assert gemm_sm100.supports_grouped(x, w, off)
    out = torch.full((rows, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    gemm_sm100.grouped_matmul_nt(x, w, off, out=out)
    s = 0
    for e, c in enumerate(counts):
        ref = x[s:s + c].float() @ w[e].float().t()
        torch.testing.assert_close(out[s:s + c].float(), ref, atol=2e-2 * max(1.0, ref.abs().max().item()) if c else 0, rtol=2e-2)
        s += c
    assert torch.isfinite(out.float()).all()


@pytest.mark.parametrize("group_m", [0, 1, 3, 8])
def test_gemm_2cta_rasterisation_groups(group_m):
    """Grouped (L2 super-block) tile order visits every tile exactly once, incl. a ragged last group and edge tiles."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    torch.manual_seed(group_m)
    M, N, K = 256 * 7 + 40, 256 * 5 + 24, 192
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    c = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    gemm_sm100.matmul_2cta(a, b, False, False, out=c, group_m=group_m)
    ref = torch.mm(a, b.t())
    assert torch.isfinite(c.float()).all()
    assert (c.float() - ref.float()).abs().max().item() < 2e-2 * ref.float().abs().max().item() + 1e-2


@pytest.mark.parametrize("shape", [(512, 384, 256), (1000, 520, 264), (6144, 4096, 8192)])
def test_gemm_2cta_accumulate_epilogue(shape):
    """EPI_ACCUM: C += A^T B (the dW accumulation of micro-batch 2..GAS) and C += A B^T."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    M, N, K = shape
    torch.manual_seed(M)
    a_km = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b_kn = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    c0 = torch.randn(M, N, device="cuda", dtype=torch.bfloat16) * 8
    c = c0.clone()
    gemm_sm100.matmul_2cta(a_km, b_kn, True, True, out=c, epi=gemm_sm100.EPI_ACCUM)
    ref = c0.float() + a_km.float().t() @ b_kn.float()
    assert (c.float() - ref).abs().max().item() < 1.5e-2 * ref.abs().max().item() + 1e-2
    a = a_km.t().contiguous()
    b = b_kn.t().contiguous()
    c = c0.clone()
    gemm_sm100.matmul_2cta(a, b, False, False, out=c, epi=gemm_sm100.EPI_ACCUM)
    assert (c.float() - ref).abs().max().item() < 1.5e-2 * ref.abs().max().item() + 1e-2


@pytest.mark.parametrize("T,H,I", [(256, 128, 128), (1000, 320, 384), (4096, 4096, 14336)])
def test_gemm_swiglu_epilogue(T, H, I):
    """EPI_SWIGLU: act = silu(x Wg^T) * (x Wu^T) from the accumulators, gate|up saved in the same pass."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    torch.manual_seed(T + I)
    x = (torch.randn(T, H, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(2 * I, H, device="cuda") * (1.0 / H**0.5)).bfloat16()
    act = torch.full((T, I), float("nan"), device="cuda", dtype=torch.bfloat16)
    gu = torch.full((T, 2 * I), float("nan"), device="cuda", dtype=torch.bfloat16)
    gemm_sm100.matmul_2cta(x, w, False, False, out=act, epi=gemm_sm100.EPI_SWIGLU, out2=gu, inter=I)
    ref_gu = x.float() @ w.float().t()
    ref_act = torch.nn.functional.silu(ref_gu[:, :I]) * ref_gu[:, I:]
    assert torch.isfinite(act.float()).all() and torch.isfinite(gu.float()).all()
    assert (gu.float() - ref_gu).abs().max().item() < 1e-2 * ref_gu.abs().max().item() + 1e-2
    assert (act.float() - ref_act).abs().max().item() < 1e-2 * ref_act.abs().max().item() + 1e-2
    # without the save
    act2 = torch.empty_like(act)
    gemm_sm100.matmul_2cta(x, w, False, False, out=act2, epi=gemm_sm100.EPI_SWIGLU, inter=I)
    assert torch.equal(act, act2)


@pytest.mark.parametrize("T,H,I", [(256, 128, 256), (1000, 320, 392), (4096, 4096, 14336)])
def test_gemm_dswiglu_epilogue(T, H, I):
    """EPI_DSWIGLU: dgate|dup = dSwiGLU(dY W_down, gate|up) with the [T, I] intermediate gradient kept in registers."""
    from deepspeed_b200.ops.kernels import gemm_sm100
    torch.manual_seed(T + I)
    dy = (torch.randn(T, H, device="cuda") * 0.5).bfloat16()
    wd = (torch.randn(H, I, device="cuda") * (1.0 / H**0.5)).bfloat16()
    gu = torch.randn(T, 2 * I, device="cuda").bfloat16()
    dgu = torch.full((T, 2 * I), float("nan"), device="cuda", dtype=torch.bfloat16)
    gemm_sm100.matmul_2cta(dy, wd, False, True, out=dgu[:, :I], epi=gemm_sm100.EPI_DSWIGLU, aux=gu, out2=dgu, inter=I)
    d_act = dy.float() @ wd.float()
    g = gu[:, :I].float().requires_grad_(True)
    u = gu[:, I:].float().requires_grad_(True)
    (torch.nn.functional.silu(g) * u).backward(d_act)
    ref = torch.cat([g.grad, u.grad], dim=1)
    assert torch.isfinite(dgu.float()).all()
    assert (dgu.float() - ref).abs().max().item() < 1.5e-2 * ref.abs().max().item() + 1e-2


@pytest.mark.parametrize("backend", ["own", "lib"])
def test_swiglu_mlp_matches_autograd(backend):
    """Fused SwiGLU MLP node (3 GEMM launches per direction, activation in the epilogues) vs plain autograd."""
    from deepspeed_b200.ops import gemm
    from deepspeed_b200.ops.linear import swiglu_mlp
    prev = gemm.get_backend()
    gemm.set_backend(backend)
    try:
        torch.manual_seed(0)
        T, H, I = 1024, 512, 1280
        x = (torch.randn(2, T // 2, H, device="cuda") * 0.5).bfloat16().requires_grad_(True)
        wg = (torch.randn(2 * I, H, device="cuda") / H**0.5).bfloat16().requires_grad_(True)
        wd = (torch.randn(H, I, device="cuda") / I**0.5).bfloat16().requires_grad_(True)
        y = swiglu_mlp(x, wg, wd)
        gy = torch.randn_like(y)
        y.backward(gy)
        xr, wgr, wdr = (t.detach().float().requires_grad_(True) for t in (x, wg, wd))
        gu = xr @ wgr.t()
        yr = (torch.nn.functional.silu(gu[..., :I]) * gu[..., I:]) @ wdr.t()
        yr.backward(gy.float())
        for got, ref in ((y, yr), (x.grad, xr.grad), (wg.grad, wgr.grad), (wd.grad, wdr.grad)):
            s = ref.float().abs().max().item()
            assert (got.float() - ref.float()).abs().max().item() < 3e-2 * s + 1e-2
    finally:
        gemm.set_backend(prev)


def test_grouped_swiglu_experts_match_bmm_reference():
    """MoE training experts: wgmma per-expert fused path vs the batched-GEMM autograd reference."""
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    torch.manual_seed(0)
    E, C, H, I = 2, 512, 256, 384
    ex = GroupedSwiGLUExperts(E, H, I).cuda().bfloat16()
    x = (torch.randn(E, C, H, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    y = ex(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().float().requires_grad_(True)
    w13, w2 = ex.w13.detach().float().requires_grad_(True), ex.w2.detach().float().requires_grad_(True)
    gu = torch.bmm(xr, w13.transpose(1, 2))
    yr = torch.bmm(torch.nn.functional.silu(gu[..., :I]) * gu[..., I:], w2.transpose(1, 2))
    yr.backward(gy.float())
    for got, ref in ((y, yr), (x.grad, xr.grad), (ex.w13.grad, w13.grad), (ex.w2.grad, w2.grad)):
        s = ref.abs().max().item()
        assert (got.float() - ref).abs().max().item() < 3e-2 * s + 1e-2
