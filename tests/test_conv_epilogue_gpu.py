"""The epilogues of the 32-channel down and up convolutions (csrc/dv_conv_tc.cu): both request the mask words before
the MMAs whose outputs they mask, and the up kernel's two consumer warpgroups take their epilogues in turn.

Through the raw C ABI, on every geometry the kernels accept (lo 16, 8, 4), with pixel counts whose last tile is ragged
(the second warpgroup's 64 rows partly or entirely past the end) and with grids smaller than the SM count: every output
against an fp64 reference, with and without the float mask and its bit words, with bias + ReLU and without.  Outputs,
bit words and channel-sum workspaces sit between sentinel words, inputs are followed by NaN, and every call runs twice
and must repeat bit for bit."""
import pytest
import torch
import torch.nn.functional as F

SENTINEL = 0x7FBADBAD   # a NaN bit pattern no kernel writes
GUARD = 256             # words of sentinel before and after each output
ACT_NONE, ACT_RELU = 0, 1
TOL = 2e-6              # of the fp64 sum of |terms|: 3xTF32 sits near 2^-22, one tf32 pass near 2^-11
SM_COUNT = 132

# (B, lo H = W): the last down tile of B = 1 and 3 at lo 4 and of B = 33 at lo 8 leaves warpgroup 1's 64 rows empty,
# B = 37 at lo 4 leaves them partly filled (up: B = 1 and 3 at lo 4 fill part of one tile of 8 images); B = 170 at
# lo 16 runs more tiles than SMs, the others fewer.
CASES = [(1, 4), (3, 4), (37, 4), (33, 8), (64, 8), (37, 16), (170, 16)]
MASKS = ["relu_bias", "float_mask", "mask_bits"]


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from disvae import _native
    return _native.lib()


def _guarded(n, dtype=torch.float32):
    """(buffer, view of n elements GUARD words in), the rest of the buffer filled with SENTINEL."""
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(dtype)


def _guards_intact(buf, n):
    return bool((buf[:GUARD] == SENTINEL).all() and (buf[GUARD + n:] == SENTINEL).all())


def _nan_after(t):
    """t's values in a buffer followed by NaN: a read past the end poisons the result."""
    buf = torch.full((t.numel() + 64,), float("nan"), device="cuda").view(torch.int32).view(t.dtype)
    buf[:t.numel()] = t.reshape(-1)
    return buf


def _ptr(t):
    return None if t is None else t.data_ptr()


def _inputs(B, H, seed):
    g = torch.Generator().manual_seed(seed)
    hi = torch.randn(B, 2 * H, 2 * H, 32, generator=g)
    lo = torch.randn(B, H, H, 32, generator=g)
    w = torch.randn(32, 32, 4, 4, generator=g) * 0.1
    bias = torch.randn(32, generator=g) * 0.1
    mask_lo = torch.randn(B, H, H, 32, generator=g)
    mask_hi = torch.randn(B, 2 * H, 2 * H, 32, generator=g)
    return hi, lo, w, bias, mask_lo, mask_hi


def _words(mask):
    """[mask > 0] per pixel as one int32 word, bit c = channel c."""
    v = ((mask > 0).to(torch.int64) << torch.arange(32, dtype=torch.int64)).sum(-1)
    return torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32)


def _ref(x_nhwc, w, bias, act, mask, transpose):
    """fp64 reference and the fp64 sum of |terms| in NHWC."""
    x = x_nhwc.double().permute(0, 3, 1, 2)
    wd = w.double()
    conv = F.conv_transpose2d if transpose else F.conv2d
    ref = conv(x, wd, stride=2, padding=1)
    terms = conv(x.abs(), wd.abs(), stride=2, padding=1)
    if bias is not None:
        ref = ref + bias.double().view(1, -1, 1, 1)
        terms = terms + bias.double().abs().view(1, -1, 1, 1)
    ref, terms = ref.permute(0, 2, 3, 1), terms.permute(0, 2, 3, 1)
    if act == ACT_RELU:
        ref = ref.clamp_min(0)
    if mask is not None:
        ref = torch.where(mask > 0, ref, torch.zeros_like(ref))
    return ref, terms


def _run(lib, op, B, H, kind, x, wp, bias, mask, out_numel, px):
    """One call on guarded buffers -> (output, bit words, channel sums or None).  mask: on the host."""
    act = ACT_RELU if kind == "relu_bias" else ACT_NONE
    b = _nan_after(bias.cuda()) if kind == "relu_bias" else None
    m = _nan_after(mask.cuda()) if kind != "relu_bias" else None
    mb = _nan_after(_words(mask).cuda()) if kind == "mask_bits" else None
    out_buf, out = _guarded(out_numel)
    bits_buf, bits = _guarded(px, torch.int32)
    stream = torch.cuda.current_stream().cuda_stream
    if op == "down":
        cs_buf, cs = _guarded(32)
        ws_bytes = lib.dv_channel_sum_workspace_bytes()
        ws_buf, ws = _guarded(ws_bytes // 4)
        rc = lib.dv_conv_down(_ptr(x), _ptr(wp), _ptr(b), _ptr(m), _ptr(out), B, H, H, 32, 0, act, _ptr(cs), _ptr(ws),
                              _ptr(mb), _ptr(bits), stream)
    else:
        rc = lib.dv_conv_up(_ptr(x), _ptr(wp), _ptr(b), _ptr(m), _ptr(out), B, H, H, 32, 0, act, _ptr(mb), _ptr(bits),
                            stream)
    torch.cuda.synchronize()
    assert rc == 0, rc
    assert _guards_intact(out_buf, out_numel) and _guards_intact(bits_buf, px), "write outside the output"
    if op == "down":
        assert _guards_intact(cs_buf, 32) and _guards_intact(ws_buf, ws_bytes // 4), "write outside the channel sums"
        return out.clone(), bits.clone(), cs.clone()
    return out.clone(), bits.clone(), None


@pytest.mark.gpu
@pytest.mark.parametrize("kind", MASKS)
@pytest.mark.parametrize("op", ["down", "up"])
@pytest.mark.parametrize("B,H", CASES, ids=["B%d-lo%d" % c for c in CASES])
def test_epilogue_against_fp64(lib, B, H, op, kind):
    from disvae import ops
    hi, lo, w, bias, mask_lo, mask_hi = _inputs(B, H, 100 * H + B)
    wp = ops.conv_pack(w.cuda(), 32)
    if op == "down":
        x, mask, out_shape = hi, mask_lo, (B, H, H, 32)
    else:
        x, mask, out_shape = lo, mask_hi, (B, 2 * H, 2 * H, 32)
    px = out_shape[0] * out_shape[1] * out_shape[2]
    out_numel = px * 32
    x_d = _nan_after(x.cuda())
    args = (lib, op, B, H, kind, x_d, wp, bias, mask, out_numel, px)
    got, bits, cs = _run(*args)
    again = _run(*args)
    assert torch.equal(got.view(torch.int32), again[0].view(torch.int32)), "not bit-identical between two calls"
    assert torch.equal(bits, again[1])
    if cs is not None:
        assert torch.equal(cs.view(torch.int32), again[2].view(torch.int32))

    act = ACT_RELU if kind == "relu_bias" else ACT_NONE
    ref, terms = _ref(x, w, bias if kind == "relu_bias" else None, act, mask if kind != "relu_bias" else None,
                      transpose=(op == "up"))
    got = got.view(out_shape).cpu().double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    ratio = (err / (TOL * terms + 1e-30)).max().item()
    print("%s B=%d lo%d %s: worst error %.3f of the bound" % (op, B, H, kind, ratio))
    assert ratio <= 1.0
    if kind != "relu_bias":
        assert (got[mask <= 0] == 0).all(), "a masked channel is not zero"
    assert torch.equal(bits.cpu(), _words(got.float()).view(-1)), "bit words are not [out > 0]"
    if cs is not None:
        s = got.sum(dim=(0, 1, 2))
        assert ((cs.cpu().double() - s).abs() <= 1e-4 * got.abs().sum(dim=(0, 1, 2)) + 1e-30).all()


def test_cases_cover_small_grids_and_ragged_tiles():
    """The case list keeps the tails and grid sizes the kernels' schedules depend on."""
    tiles = {(B, H): -(-B * H * H // 128) for B, H in CASES}
    assert any(t < SM_COUNT for t in tiles.values()) and any(t > SM_COUNT for t in tiles.values())
    tails = {(B, H): (B * H * H) % 128 for B, H in CASES}
    assert any(0 < r <= 64 for r in tails.values())                # warpgroup 1's rows empty
    assert any(r > 64 for r in tails.values())                     # ... partly filled
