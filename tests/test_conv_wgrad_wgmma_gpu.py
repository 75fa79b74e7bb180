"""The 32-channel weight-gradient convolution (wgmma kernel of dv_conv_tc.cu, with the lo tile transposed and split into
hi/lo planes once per tile) against fp64: the shapes of the training steps, ragged batches that leave a partial last
tile and a short last CTA, the decoder's use (lo = gradient of a ConvTranspose2d output) and a lo tile with rows of
exact zeros beside values up to 1e4.  Every case is run twice and must repeat bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TOL = 4e-6          # of the output scale: fp32-grade (single-pass tf32 lands near 5e-4)

# batch per GPU of c2, c3 and c5 at lo 16, 8 and 4; then batches whose last 128-pixel tile is partial (37 at lo 4,
# 33 at lo 8) or whose last CTA gets fewer tiles than the others (170 and 600 at lo 16)
SHAPES = [(B, H) for B in (1024, 512, 256) for H in (16, 8, 4)]
RAGGED = [(37, 4), (33, 8), (170, 16), (600, 16)]


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def rel_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def check_wgrad(hi, lo):
    """hi [B, 32, 2H, 2H], lo [B, 32, H, H] on the host: dw and db of the kernel against fp64, twice."""
    from disvae import ops
    B, H = lo.shape[0], lo.shape[2]
    hi_d, lo_d = nhwc(hi).to(DEV), nhwc(lo).to(DEV)
    dw, db = ops.conv_wgrad(lo_d, hi_d, B, H, H, 32, 0, True)
    want_dw = torch.nn.grad.conv2d_weight(hi.double(), (32, 32, 4, 4), lo.double(), stride=2, padding=1)
    want_db = lo.double().sum((0, 2, 3))
    assert rel_err(dw, want_dw) <= TOL
    assert rel_err(db, want_db) <= TOL
    dw2, db2 = ops.conv_wgrad(lo_d, hi_d, B, H, H, 32, 0, True)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


@pytest.mark.parametrize("B,H", SHAPES + RAGGED)
def test_conv_wgrad32_vs_fp64(B, H):
    torch.manual_seed(7 * B + H)
    check_wgrad(torch.randn(B, 32, 2 * H, 2 * H), torch.randn(B, 32, H, H))


def test_conv_wgrad32_of_conv_transpose_gradient():
    """The decoder's use: the upsampling layer's weight gradient is the same correlation with the roles swapped, lo =
    the layer's input and hi = the gradient of its output.  Against autograd in fp64."""
    from disvae import ops
    torch.manual_seed(3)
    B, H = 96, 8
    x = torch.randn(B, 32, H, H, dtype=torch.float64)
    w = (torch.randn(32, 32, 4, 4, dtype=torch.float64) * 0.1).requires_grad_()
    g = torch.randn(B, 32, 2 * H, 2 * H, dtype=torch.float64)
    F.conv_transpose2d(x, w, None, stride=2, padding=1).backward(g)
    dw, _ = ops.conv_wgrad(nhwc(x.float()).to(DEV), nhwc(g.float()).to(DEV), B, H, H, 32, 0, False)
    want = torch.nn.grad.conv2d_weight(g.float().double(), (32, 32, 4, 4), x.float().double(), stride=2, padding=1)
    assert rel_err(w.grad, want) <= TOL          # the identity the decoder relies on (fp32 rounding of the inputs only)
    assert rel_err(dw, want) <= TOL
    dw2, _ = ops.conv_wgrad(nhwc(x.float()).to(DEV), nhwc(g.float()).to(DEV), B, H, H, 32, 0, False)
    assert torch.equal(dw, dw2)


def test_conv_wgrad32_zero_rows_and_large_values():
    """Both ends of the hi/lo split of the lo tile: pixels whose 32 channels are exactly zero (as behind a ReLU mask)
    and magnitudes from 1e-4 to 1e4 in the same tile."""
    torch.manual_seed(4)
    B, H = 64, 8
    hi = torch.randn(B, 32, 2 * H, 2 * H)
    lo = torch.randn(B, 32, H, H) * 10.0 ** torch.randint(-4, 5, (B, 32, H, H)).float()
    lo = lo * (torch.rand(B, 1, H, H) > 0.4)     # whole pixels zeroed: zero rows of the [pixel][channel] tile
    assert (lo.abs().amax(1) == 0).any() and lo.abs().max() > 1e4
    check_wgrad(hi, lo)
