"""Kernel objects / module layer of the ragged engine on the device: the sm_90a kernels behind them must agree with the
host (plain torch fp32) path of the very same objects."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepspeed_b200.inference.v2.inference_utils import ActivationType, DtypeEnum, NormTypeEnum  # noqa: E402
from deepspeed_b200.inference.v2.kernels.core_ops import (BlasLibLinear, CUDABiasActivation, CUDAFPPreLN,  # noqa: E402
                                                          CUDAGatedActivation, CUDARMSPreNorm)
from deepspeed_b200.inference.v2.kernels.ragged_ops import (BlockedFlashAttn, BlockedRotaryEmbeddings, MoEGather,  # noqa: E402
                                                            MoEScatter, RaggedLogitsGather, RaggedTopKGating)
from deepspeed_b200.inference.v2.modules import heuristics as H  # noqa: E402
from deepspeed_b200.inference.v2.modules.configs import DSLinearConfig, DSMoEConfig, DSNormConfig  # noqa: E402
from deepspeed_b200.utils.types import ActivationFuncType  # noqa: E402


def _close(a, b, tol=3e-2):
    a, b = a.float().cpu(), b.float().cpu()
    assert (a - b).abs().max() <= tol * max(1.0, b.abs().max().item()), (a - b).abs().max()


def test_core_ops_device_vs_host():
    torch.manual_seed(0)
    x, y = torch.randn(64, 1024), torch.randn(64, 1024)
    g, b = torch.rand(1024) + 0.5, torch.randn(1024)
    for make, args in ((lambda dt: CUDAFPPreLN(1024, dt), (g, b)), (lambda dt: CUDARMSPreNorm(1024, dt), (g, ))):
        ref = make(torch.float32)(torch.empty_like(x), torch.empty_like(x), x.clone(), y.clone(), *args)
        dx, dy = x.cuda().bfloat16(), y.cuda().bfloat16()
        out = make(torch.bfloat16)(torch.empty_like(dx), torch.empty_like(dx), dx, dy, *[a.cuda().bfloat16() for a in args])
        _close(out[0], ref[0])
        _close(out[1], ref[1])
    a = x.clone()
    CUDABiasActivation(1024, torch.float32, ActivationFuncType.GELU)(a, b)
    da = x.cuda().bfloat16()
    CUDABiasActivation(1024, torch.bfloat16, ActivationFuncType.GELU)(da, b.cuda().bfloat16())
    _close(da, a)
    ref = CUDAGatedActivation(1024, torch.float32, ActivationFuncType.GATED_SILU)(torch.empty(64, 512), x)
    out = CUDAGatedActivation(1024, torch.bfloat16, ActivationFuncType.GATED_SILU)(torch.empty(64, 512, device="cuda", dtype=torch.bfloat16),
                                                                                  x.cuda().bfloat16())
    _close(out, ref)
    w = torch.randn(256, 1024) * 0.05
    out = BlasLibLinear(torch.bfloat16)(torch.empty(64, 256, device="cuda", dtype=torch.bfloat16), x.cuda().bfloat16(), w.cuda().bfloat16())
    _close(out, x @ w.t(), 5e-2)


def test_ragged_attention_and_gather_device_vs_host():
    torch.manual_seed(0)
    hq, hkv, d, bs = 8, 2, 128, 128
    lens = [200, 37, 1]
    T = sum(lens)
    seq_of = torch.cat([torch.full((n, ), i, dtype=torch.int32) for i, n in enumerate(lens)])
    pos_of = torch.cat([torch.arange(n, dtype=torch.int32) for n in lens])
    bt = torch.tensor([[0, 1], [2, 3], [4, 5]], dtype=torch.int32)
    qkv = torch.randn(T, (hq + 2 * hkv) * d) * 0.5

    def run(dev, dt):
        cache = torch.zeros(6, bs, 2, hkv, d, device=dev, dtype=dt)
        q = qkv.to(dev, dt).clone()
        BlockedRotaryEmbeddings(d, hq, hkv, dt, d, 10000.0, max_positions=512)(cache, q, seq_of.to(dev), pos_of.to(dev), bt.to(dev), bs)
        out = torch.empty(T, hq * d, device=dev, dtype=dt)
        BlockedFlashAttn(d, dt)(out, q, cache, seq_of.to(dev), pos_of.to(dev), bt.to(dev), hq, hkv, bs)
        last = torch.empty(3, hq * d, device=dev, dtype=dt)
        RaggedLogitsGather(hq * d, dt)(last, out, torch.tensor([199, 236, 237], dtype=torch.int32, device=dev))
        return out, last

    ref, ref_last = run("cpu", torch.float32)
    out, last = run("cuda", torch.bfloat16)
    _close(out, ref)
    _close(last, ref_last)


def test_moe_module_device_vs_host():
    torch.manual_seed(0)
    x = torch.randn(96, 256) * 0.5
    gw, w1, w2 = torch.randn(8, 256) * 0.2, torch.randn(8, 2 * 512, 256) * 0.05, torch.randn(8, 256, 512) * 0.05

    def run(dev, dt, enum):
        moe = H.instantiate_moe(DSMoEConfig(model_dim=256, intermediate_features=512, n_experts=8, top_k=2, input_dtype=enum,
                                            output_dtype=enum, activation=ActivationType.SiGLU, normalize_scores=True))
        return moe(x.to(dev, dt), gw.to(dev, dt), w1.to(dev, dt), w2.to(dev, dt))

    ref = run("cpu", torch.float32, DtypeEnum.fp32)
    out = run("cuda", torch.bfloat16, DtypeEnum.bf16)
    # routing of near-tied tokens may differ under bf16 logits: compare the bulk
    err = (out.float().cpu() - ref).abs().max(dim=1).values
    assert (err < 0.05).float().mean() > 0.95, err.topk(5).values


def test_linear_and_norm_modules_on_device():
    torch.manual_seed(0)
    bf = DtypeEnum.bf16
    lin = H.instantiate_linear(DSLinearConfig(in_channels=512, out_channels=256, activation=ActivationType.GEGLU, input_dtype=bf,
                                              output_dtype=bf))
    x, w = torch.randn(32, 512), torch.randn(512, 512) * 0.05
    y = lin(x.cuda().bfloat16(), w.cuda().bfloat16())
    h = x @ w.t()
    _close(y, torch.nn.functional.gelu(h[:, :256]) * h[:, 256:], 5e-2)
    qlin = H.instantiate_linear(DSLinearConfig(in_channels=512, out_channels=512, input_dtype=bf, output_dtype=bf, quantization_mode="int4"))
    qw = qlin.transform_param(w.cuda().bfloat16())
    _close(qlin(x[:8].cuda().bfloat16(), qw), x[:8] @ qw.dequantize().float().cpu().t(), 5e-2)
    pre = H.instantiate_pre_norm(DSNormConfig(type=NormTypeEnum.RMSNorm, channels=512, residual_dtype=bf, input_dtype=bf, output_dtype=bf))
    res, delta, g = torch.randn(32, 512), torch.randn(32, 512), torch.rand(512) + 0.5
    r2, hid = pre(res.cuda().bfloat16(), delta.cuda().bfloat16(), g.cuda().bfloat16())
    want = res + delta
    _close(r2, want)
    _close(hid, want * torch.rsqrt(want.pow(2).mean(-1, keepdim=True) + 1e-5) * g)
