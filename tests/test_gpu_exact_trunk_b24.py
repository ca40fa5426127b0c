"""Exact-mode 3x3 trunk convolutions (igemm_kernel<256, SPLIT>) at the batch the benchmark runs them at, B = 24: against float64 on
a slice of items and output channels, held to the accumulation bar of
test_gpu_exact.py::test_exact_trunk_conv_k9216_accumulation_error (2.5e-5 of the output scale), and independent of the batch
size bit for bit (a tile's accumulation order does not depend on how many tiles the launch has)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"
BAR = 2.5e-5


@pytest.mark.parametrize("C", [1024, 512], ids=["res2_trunk_1024", "res3_512"])
def test_exact_trunk_conv_at_b24_vs_float64_and_batch_independent(C):
    from rendernet_b200 import ops
    B, H, W = 24, 64, 64
    g = torch.Generator(device="cpu").manual_seed(C)
    x = torch.randn(B, H, W, C, generator=g) * 3
    w = (torch.rand(3, 3, C, C, generator=g) * 2 - 1) * (6.0 / (9 * 2 * C)) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    L = ops.pack_conv("conv2d", w, b, None, device=dev, fmt=2)

    def run(xin):
        y = ops.conv2d(ops.cast_to_16(xin.to(dev), fmt=2), L, want16=False, want32=True)
        torch.cuda.synchronize()
        return y

    y = run(x)
    items, co = [0, 13, 23], slice(0, 64)
    ref = F.conv2d(x[items].double().permute(0, 3, 1, 2), w[:, :, :, co].double().permute(3, 2, 0, 1), b[co].double(),
                   padding=1).permute(0, 2, 3, 1)
    s = float(ref.abs().max())
    err = float((y[items][..., co].double().cpu() - ref).abs().max())
    print(f"3x3 {C}->{C} B=24 exact vs float64 (items {items}, 64 channels): {err / s:.2e} of scale")
    assert err <= BAR * s

    assert torch.equal(run(x[:8]), y[:8])
    for i in items:
        assert torch.equal(run(x[i:i + 1]), y[i:i + 1]), i
