"""torch.autograd.Function wrappers over the C ABI (include/disvae_b200.h).

PyTorch is plumbing here: it owns device memory, streams and the autograd tape between the
big nodes (encoder, decoder, discriminator, loss heads).  Every FLOP of the hot path runs in
libdisvae_b200.so.  All functions require CUDA fp32 tensors and raise otherwise.
"""
import contextlib
import os as _os

import torch
from torch.autograd import Function

from . import _native as N
from ._native import ACT_LEAKY, ACT_NONE, ACT_RELU, ACT_SIGMOID, call, ptr, stream

LO_CH = 32
FLAT = 512          # 32 channels x 4 x 4  (encoders.py:63, decoders.py:55)
DISC_SLOPE = 0.2    # discriminator.py:10

# ---------------------------------------------------------------------------------------
# persistent, zero-initialised scratch (kernels that use a "last block done" counter leave
# it at zero, so one buffer per device can be reused across calls on the same stream)
#
# Every per-process resource below -- this scratch, the beta-TCVAE workspaces and the weight-gradient side stream -- is
# keyed by the current owner as well as the device.  The owner is None except inside `owner(token)`: disvae.sweep runs
# each member's eager steps and graph capture under its own token, so members whose graphs replay concurrently never
# share a split-K partial buffer, a "last block done" counter or a side stream.
# ---------------------------------------------------------------------------------------
_persist = {}
_in_graph = set()      # keys of _persist whose current buffer was handed out during a CUDA-graph capture
_retired = {}          # owner -> such buffers after a larger one replaced them: the graph still reads their addresses
_owner = None


@contextlib.contextmanager
def owner(token):
    """Kernels called inside use the scratch, workspaces and side stream of `token` (any hashable; None = the
    process-wide set a lone Trainer uses)."""
    global _owner
    old, _owner = _owner, token
    try:
        yield
    finally:
        _owner = old


def release(token):
    """Drop the scratch, workspaces and side stream of owner `token` (once nothing that uses them can run again)."""
    for table in (_persist, _bt_pool, _side_streams):
        for k in [k for k in table if k[-1] == token]:
            del table[k]
    _in_graph.difference_update([k for k in _in_graph if k[-1] == token])
    _retired.pop(token, None)


def _persistent(key, nbytes, device, alloc):
    k = (key, device.index, _owner)
    buf = _persist.get(k)
    if buf is None or buf.numel() * 4 < nbytes:
        # A buffer only eager kernels used is freed: each key is used on one stream, and the caching allocator hands the
        # block only to later work on that stream.  One a captured graph baked in must outlive the graph: kept.
        if k in _in_graph:
            _retired.setdefault(_owner, []).append(buf)
            _in_graph.discard(k)
        buf = alloc((nbytes + 3) // 4, dtype=torch.float32, device=device)
        _persist[k] = buf
    if torch.cuda.is_current_stream_capturing():
        _in_graph.add(k)
    return buf


def _zero_ws(key, nbytes, device):
    return _persistent(key, nbytes, device, torch.zeros)


def _scratch(key, nbytes, device):
    """Non-zeroed scratch, grown on demand (channel sums, wgrad partials)."""
    return _persistent(key, nbytes, device, torch.empty)


def _new(shape, like):
    return torch.empty(shape, dtype=torch.float32, device=like.device)


# Activation trace for the parity checks (same_branch.py next to the CPU reference restatement): while a list is installed, the three network nodes append
# (name, tensor) for every (Leaky)ReLU output they produce -- the on/off pattern a flip-robust gradient comparison needs.
# None in production: one `is not None` test per layer.
_trace = None


def start_trace():
    global _trace
    _trace = []
    return _trace


def stop_trace():
    global _trace
    t, _trace = _trace, None
    return t


def _note(name, t):
    if _trace is not None:
        _trace.append((name, t))


# ---------------------------------------------------------------------------------------
# thin functional layer (one C call each) -- also what the per-kernel parity tests use
# ---------------------------------------------------------------------------------------
def conv_pack(w, CH):
    wp = _new((N.lib().dv_conv_packed_floats(CH),), w)
    call("dv_conv_pack_weights", ptr(w), ptr(wp), CH, stream())
    return wp


def conv_pack_multi(weights, chans):
    """Packed operands of every conv layer of a network node in ONE launch -> list of packed buffers."""
    import ctypes
    L = N.lib()
    n = len(weights)
    packs = [_new((L.dv_conv_packed_floats(ch),), w) for w, ch in zip(weights, chans)]
    arr_p = ctypes.c_void_p * n
    call("dv_conv_pack_multi", n, arr_p(*[w.data_ptr() for w in weights]), arr_p(*[p.data_ptr() for p in packs]),
         (ctypes.c_int * n)(*chans), stream())
    return packs


def conv_down(hi, wp, bias, mask, B, H, W, CH, nchw, act, want_colsum=False, mask_bits=None, want_bits=False):
    """-> lo; with want_colsum also the channel sums of lo (summed in the kernel's epilogue); with want_bits also
    [lo > 0] as one int32 word per pixel (the mask_bits of the backward pass through the ReLU after this layer)."""
    lo = _new((B, H, W, LO_CH), hi)
    cs = ws = None
    if want_colsum:
        cs = _new((LO_CH,), hi)
        ws = _scratch("chansum", N.lib().dv_channel_sum_workspace_bytes(), hi.device)
    bits = torch.empty((B, H, W), dtype=torch.int32, device=hi.device) if want_bits else None
    call("dv_conv_down", ptr(hi), ptr(wp), ptr(bias), ptr(mask), ptr(lo), B, H, W, CH, nchw, act, ptr(cs), ptr(ws),
         ptr(mask_bits), ptr(bits), stream(), tag="[H=%d,CH=%d]%s" % (H, CH, "+mask" if mask is not None else ""))
    out = (lo,) + ((cs,) if want_colsum else ()) + ((bits,) if want_bits else ())
    return out if len(out) > 1 else lo


def conv_up(lo, wp, bias, mask, B, H, W, CH, nchw, act, mask_bits=None, want_bits=False):
    hi = _new((B, CH, 2 * H, 2 * W) if nchw else (B, 2 * H, 2 * W, CH), lo)
    bits = torch.empty((B, 2 * H, 2 * W), dtype=torch.int32, device=lo.device) if want_bits else None
    call("dv_conv_up", ptr(lo), ptr(wp), ptr(bias), ptr(mask), ptr(hi), B, H, W, CH, nchw, act, ptr(mask_bits), ptr(bits),
         stream(), tag="[H=%d,CH=%d]%s" % (H, CH, "+mask" if mask is not None else ""))
    return (hi, bits) if want_bits else hi


def conv_wgrad(lo, hi, B, H, W, CH, nchw, want_dbias_lo):
    L = N.lib()
    nbytes = L.dv_conv_wgrad_workspace_bytes(B, H, W, CH)
    ws = _scratch("wgrad", nbytes, lo.device)
    dw = _new((LO_CH, CH, 4, 4), lo)
    db = _new((LO_CH,), lo) if want_dbias_lo else None
    call("dv_conv_wgrad", ptr(lo), ptr(hi), ptr(dw), ptr(db), ptr(ws), nbytes, B, H, W, CH, nchw, stream(),
         tag="[H=%d,CH=%d]" % (H, CH))
    return dw, db


def channel_sum(x, rows, C, nchw, hw):
    ws = _scratch("chansum", N.lib().dv_channel_sum_workspace_bytes(), x.device)
    out = _new((C,), x)
    call("dv_channel_sum", ptr(x), ptr(out), rows, C, nchw, hw, ptr(ws), stream())
    return out


def flat_transpose(src, B, to_nhwc):
    dst = torch.empty_like(src)
    call("dv_flat_transpose", ptr(src), ptr(dst), B, LO_CH, 16, int(to_nhwc), stream())
    return dst


def act_bwd_chansum(dy, y, act, slope=0.0):
    """g = dy * act'(y) over an NCHW tensor and, from the same pass, the per-channel sums of g."""
    B, C = y.shape[0], y.shape[1]
    hw = y.numel() // (B * C)
    g = torch.empty_like(y)
    cs = _new((C,), y)
    ws = _scratch("chansum", N.lib().dv_channel_sum_workspace_bytes(), y.device)
    call("dv_act_bwd_chansum", ptr(dy), ptr(y), ptr(g), B, C, hw, act, slope, ptr(cs), ptr(ws), stream())
    return g, cs


def u8_to_f32(src, out=None):
    """uint8 CUDA tensor -> float32 / 255 (ToTensor on the device); `out` = preallocated float32 tensor of the same shape."""
    if not src.is_cuda or src.dtype != torch.uint8:
        raise RuntimeError("disvae_b200.u8_to_f32 expects a CUDA uint8 tensor, got %s on %s" % (src.dtype, src.device))
    src = _c(src)
    if out is None:
        out = torch.empty(src.shape, dtype=torch.float32, device=src.device)
    call("dv_u8_to_f32", src.data_ptr(), ptr(out), src.numel(), stream())
    return out


def gather_u8_to_f32(src, idx, out=None):
    """Rows src[idx] of a CUDA uint8 tensor [N, ...] as float32 / 255 (ToTensor on the device) in one launch;
    idx = CUDA int64 indices in [0, N), repeats allowed; `out` = preallocated float32 [len(idx), ...]."""
    if not src.is_cuda or src.dtype != torch.uint8:
        raise RuntimeError("disvae_b200.gather_u8_to_f32 expects a CUDA uint8 tensor, got %s on %s" % (src.dtype, src.device))
    if not idx.is_cuda or idx.dtype != torch.int64 or idx.dim() != 1:
        raise RuntimeError("disvae_b200.gather_u8_to_f32 expects 1-d CUDA int64 indices, got %s %s on %s"
                           % (idx.dtype, tuple(idx.shape), idx.device))
    src, idx = _c(src), _c(idx)
    if out is None:
        out = torch.empty((idx.numel(),) + tuple(src.shape[1:]), dtype=torch.float32, device=src.device)
    call("dv_gather_u8_to_f32", src.data_ptr(), idx.data_ptr(), idx.numel(), src[0].numel(), ptr(out), stream())
    return out


def index_permutation(n, seed, offset_dev, out=None):
    """Philox-keyed permutation of [0, n) as CUDA int64 (the order dv_permute_dims_rows draws for one dimension);
    reads the counter offset from the device tensor `offset_dev` and advances it by n."""
    device = offset_dev.device
    if out is None:
        out = torch.empty(n, dtype=torch.int64, device=device)
    nbytes = N.lib().dv_index_permutation_workspace_bytes(n)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device) if nbytes else None
    call("dv_index_permutation", n, seed, ptr(offset_dev), ptr(out), ptr(ws), stream())
    return out


def act_bwd(dy, y, act, slope=0.0):
    g = torch.empty_like(y)
    call("dv_act_bwd", ptr(dy), ptr(y), ptr(g), y.numel(), act, slope, stream())
    return g


def linear_pack_multi(weights):
    """Operand planes of every weight matrix of a network node in ONE launch -> list of packed buffers (pass them to
    linear_fwd / linear_dgrad as `packed=`)."""
    import ctypes
    L = N.lib()
    n = len(weights)
    packs = [_new((L.dv_linear_packed_floats(w.shape[0], w.shape[1]),), w) for w in weights]
    arr_p = ctypes.c_void_p * n
    arr_i = ctypes.c_int * n
    call("dv_linear_pack_multi", n, arr_p(*[w.data_ptr() for w in weights]), arr_p(*[p.data_ptr() for p in packs]),
         arr_i(*[w.shape[0] for w in weights]), arr_i(*[w.shape[1] for w in weights]), stream())
    return packs


def linear_fwd(x, w, b, act, slope=0.0, packed=None):
    M, K = x.shape
    Nn = w.shape[0]
    y = _new((M, Nn), x)
    if packed is not None:
        call("dv_linear_fwd_packed", ptr(x), ptr(w), ptr(packed), ptr(b), ptr(y), M, Nn, K, act, slope, stream())
        return y
    nbytes = N.lib().dv_linear_fwd_workspace_bytes(M, Nn, K)
    ws = _scratch("lin_pack", nbytes, x.device) if nbytes else None
    call("dv_linear_fwd", ptr(x), ptr(w), ptr(b), ptr(y), M, Nn, K, act, slope, ptr(ws), stream())
    return y


def linear_dgrad(g, w, mask_src, act, slope=0.0, packed=None):
    M, Nn = g.shape
    K = w.shape[1]
    dx = _new((M, K), g)
    if packed is not None:
        call("dv_linear_dgrad_packed", ptr(g), ptr(w), ptr(packed), ptr(mask_src), ptr(dx), M, Nn, K, act, slope, stream())
        return dx
    nbytes = N.lib().dv_linear_dgrad_workspace_bytes(M, Nn, K)
    ws = _scratch("lin_pack", nbytes, g.device) if nbytes else None
    call("dv_linear_dgrad", ptr(g), ptr(w), ptr(mask_src), ptr(dx), M, Nn, K, act, slope, ptr(ws), stream())
    return dx


def linear_wgrad(g, x, want_bias=True):
    M, Nn = g.shape
    K = x.shape[1]
    dw = _new((Nn, K), g)
    db = _new((Nn,), g) if want_bias else None
    nbytes = N.lib().dv_linear_wgrad_workspace_bytes(M, Nn, K)
    ws = _scratch("lin_wgrad", nbytes, g.device) if nbytes else None
    call("dv_linear_wgrad", ptr(g), ptr(x), ptr(dw), ptr(db), M, Nn, K, ptr(ws), stream())
    return dw, db


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


# ---------------------------------------------------------------------------------------
# Weight-gradient lane: in a backward pass the weight gradient of a layer and the input gradient that continues the
# chain are independent.  The MLP layers and the 4x4 / 8x8 conv layers occupy a fraction of the SMs for a short time each
# (launch-latency bound), so their weight-gradient kernels run on a second stream beside the dgrad chain and are joined
# at the end of the node's backward.  Works inside CUDA-graph capture (fork/join from the capturing stream become graph
# dependencies).  Tensors read on the side stream are kept alive until the join, so the caching allocator cannot hand
# their memory to the main stream meanwhile.  DISVAE_SIDE_STREAM=0 switches it off (same kernels, same results).
# ---------------------------------------------------------------------------------------
_side_streams = {}


class _WgradLane:
    def __init__(self, device):
        self.enabled = _os.environ.get("DISVAE_SIDE_STREAM", "1") != "0"
        self.keep = []
        if self.enabled:
            self.main = torch.cuda.current_stream(device)
            key = (device.index, _owner)
            side = _side_streams.get(key)
            if side is None:
                side = _side_streams[key] = torch.cuda.Stream(device)
            self.side = side

    def run(self, fn, *reads):
        """fn() on the side stream after everything enqueued on the main stream so far; `reads` = its input tensors."""
        if not self.enabled:
            return fn()
        self.side.wait_stream(self.main)
        with torch.cuda.stream(self.side):
            out = fn()
        self.keep.extend(reads)
        return out

    def join(self):
        if self.enabled:
            self.main.wait_stream(self.side)
            self.keep.clear()


# ---------------------------------------------------------------------------------------
# Burgess encoder (disvae/models/encoders.py:69-89) as ONE autograd node
# ---------------------------------------------------------------------------------------
class EncoderFn(Function):
    """x[B,C,S,S] -> mu_logvar[B,2z].  params = (conv w,b) * n_conv + (lin w,b) * 3."""

    @staticmethod
    def forward(ctx, x, n_conv, *params):
        N.require_cuda_f32(x, *params)
        x = _c(x)
        params = [_c(p) for p in params]
        B, C, S, _ = x.shape
        convs = [(params[2 * i], params[2 * i + 1]) for i in range(n_conv)]
        lins = [(params[2 * n_conv + 2 * i], params[2 * n_conv + 2 * i + 1]) for i in range(3)]
        # operand planes of the three linear layers (both directions) in one launch, on the side stream: it runs beside
        # the convolutions below and is joined before the first linear layer
        lane = _WgradLane(x.device)
        lpk = lane.run(lambda: linear_pack_multi([w for w, _ in lins]), *[w for w, _ in lins])
        acts = []
        packed = conv_pack_multi([w for w, _ in convs], [C] + [LO_CH] * (n_conv - 1))
        hi, CH, nchw, H = x, C, 1, S // 2
        bits = []                    # [act > 0] of every layer but the last, one word per pixel: the dgrad masks
        for (w, b), wp in zip(convs, packed):
            if len(acts) < n_conv - 1:
                lo, bw = conv_down(hi, wp, b, None, B, H, H, CH, nchw, ACT_RELU, want_bits=True)
                bits.append(bw)
            else:
                lo = conv_down(hi, wp, b, None, B, H, H, CH, nchw, ACT_RELU)
            _note("encoder.conv%d" % len(acts), lo)
            acts.append(lo)
            hi, CH, nchw, H = lo, LO_CH, 0, H // 2
        flat = flat_transpose(acts[-1].view(B, FLAT), B, to_nhwc=False)          # -> [B, 32*4*4] in NCHW order
        lane.join()
        h1 = linear_fwd(flat, lins[0][0], lins[0][1], ACT_RELU, packed=lpk[0])
        h2 = linear_fwd(h1, lins[1][0], lins[1][1], ACT_RELU, packed=lpk[1])
        ml = linear_fwd(h2, lins[2][0], lins[2][1], ACT_NONE, packed=lpk[2])
        _note("encoder.lin1", h1)
        _note("encoder.lin2", h2)
        ctx.n_conv = n_conv
        ctx.save_for_backward(x, flat, h1, h2, *acts, *packed, *bits, *params, *lpk)
        return ml

    @staticmethod
    def backward(ctx, g_ml):
        n_conv = ctx.n_conv
        saved = ctx.saved_tensors
        x, flat, h1, h2 = saved[:4]
        acts = saved[4:4 + n_conv]
        packed = saved[4 + n_conv:4 + 2 * n_conv]
        bits = saved[4 + 2 * n_conv:4 + 3 * n_conv - 1]
        params = saved[4 + 3 * n_conv - 1:-3]
        lpk = saved[-3:]
        lins = [(params[2 * n_conv + 2 * i], params[2 * n_conv + 2 * i + 1]) for i in range(3)]
        B, C, S, _ = x.shape
        g = _c(g_ml)
        lane = _WgradLane(g.device)
        dlw3, dlb3 = lane.run(lambda: linear_wgrad(g, h2), g, h2)
        g2 = linear_dgrad(g, lins[2][0], h2, ACT_RELU, packed=lpk[2])
        dlw2, dlb2 = lane.run(lambda: linear_wgrad(g2, h1), g2, h1)
        g1 = linear_dgrad(g2, lins[1][0], h1, ACT_RELU, packed=lpk[1])
        dlw1, dlb1 = lane.run(lambda: linear_wgrad(g1, flat), g1, flat)
        gflat = linear_dgrad(g1, lins[0][0], flat, ACT_RELU, packed=lpk[0])      # masked by the last conv's ReLU
        g_lo = flat_transpose(gflat, B, to_nhwc=True)
        conv_grads = [None] * (2 * n_conv)
        dx = None
        for l in range(n_conv - 1, -1, -1):
            H = S >> (l + 1)
            if l > 0:
                dw, db = lane.run(lambda gl=g_lo, a=acts[l - 1], H=H: conv_wgrad(gl, a, B, H, H, LO_CH, 0, True), g_lo, acts[l - 1])
                g_lo = conv_up(g_lo, packed[l], None, acts[l - 1], B, H, H, LO_CH, 0, ACT_NONE, mask_bits=bits[l - 1])
            else:
                dw, db = lane.run(lambda gl=g_lo, H=H: conv_wgrad(gl, x, B, H, H, C, 1, True), g_lo, x)
                if ctx.needs_input_grad[0]:
                    dx = conv_up(g_lo, packed[0], None, None, B, H, H, C, 1, ACT_NONE)
            conv_grads[2 * l], conv_grads[2 * l + 1] = dw, db
        lane.join()
        return (dx, None, *conv_grads, dlw1, dlb1, dlw2, dlb2, dlw3, dlb3)


# ---------------------------------------------------------------------------------------
# Burgess decoder (disvae/models/decoders.py:67-84) as ONE autograd node
# ---------------------------------------------------------------------------------------
class DecoderFn(Function):
    """z[B,D] -> recon[B,C,S,S].  params = (lin w,b) * 3 + (convT w,b) * n_convT."""

    @staticmethod
    def forward(ctx, z, n_convT, n_chan, *params):
        N.require_cuda_f32(z, *params)
        z = _c(z)
        params = [_c(p) for p in params]
        B = z.shape[0]
        lins = [(params[2 * i], params[2 * i + 1]) for i in range(3)]
        convTs = [(params[6 + 2 * i], params[6 + 2 * i + 1]) for i in range(n_convT)]
        lpk = linear_pack_multi([w for w, _ in lins])
        h1 = linear_fwd(z, lins[0][0], lins[0][1], ACT_RELU, packed=lpk[0])
        h2 = linear_fwd(h1, lins[1][0], lins[1][1], ACT_RELU, packed=lpk[1])
        h3 = linear_fwd(h2, lins[2][0], lins[2][1], ACT_RELU, packed=lpk[2])     # [B,512] == view(B,32,4,4)
        _note("decoder.lin1", h1)
        _note("decoder.lin2", h2)
        _note("decoder.lin3", h3)
        lo = flat_transpose(h3, B, to_nhwc=True).view(B, 4, 4, LO_CH)
        acts, bits = [lo], []        # bits[t] = [acts[t + 1] > 0], one word per pixel: the mask of convT t+1's input gradient
        packed = conv_pack_multi([w for w, _ in convTs], [LO_CH] * (n_convT - 1) + [n_chan])
        H = 4
        for t, (w, b) in enumerate(convTs):
            last = (t == n_convT - 1)
            CH = n_chan if last else LO_CH
            wp = packed[t]
            if last:
                hi = conv_up(lo, wp, b, None, B, H, H, CH, 1, ACT_SIGMOID)
            else:
                hi, bw = conv_up(lo, wp, b, None, B, H, H, CH, 0, ACT_RELU, want_bits=True)
                bits.append(bw)
                _note("decoder.convT%d" % t, hi)
                acts.append(hi)
            lo, H = hi, 2 * H
        recon = lo
        ctx.n_convT, ctx.n_chan = n_convT, n_chan
        ctx.save_for_backward(z, h1, h2, recon, *acts, *packed, *bits, *params, *lpk)
        return recon

    @staticmethod
    def backward(ctx, d_recon):
        n_convT, C = ctx.n_convT, ctx.n_chan
        saved = ctx.saved_tensors
        z, h1, h2, recon = saved[:4]
        acts = saved[4:4 + n_convT]                 # acts[t] = input of convT t (NHWC)
        packed = saved[4 + n_convT:4 + 2 * n_convT]
        bits = saved[4 + 2 * n_convT:4 + 3 * n_convT - 1]
        params = saved[4 + 3 * n_convT - 1:-3]
        lpk = saved[-3:]
        lins = [(params[2 * i], params[2 * i + 1]) for i in range(3)]
        B = z.shape[0]
        S = recon.shape[-1]
        # sigmoid backward of the output layer fused with its bias gradient (the sum of the result over pixels)
        g_hi, db = act_bwd_chansum(_c(d_recon), recon, ACT_SIGMOID)                # NCHW, C channels
        convT_grads = [None] * (2 * n_convT)
        lane = _WgradLane(g_hi.device)
        for t in range(n_convT - 1, -1, -1):
            last = (t == n_convT - 1)
            H = 4 << t                                   # input resolution of convT t
            CH, nchw = (C, 1) if last else (LO_CH, 0)
            dw, _ = lane.run(lambda a=acts[t], gh=g_hi, H=H, CH=CH, nchw=nchw: conv_wgrad(a, gh, B, H, H, CH, nchw, False),
                             acts[t], g_hi)
            convT_grads[2 * t], convT_grads[2 * t + 1] = dw, db
            # input gradient, masked by acts[t] > 0; for t > 0 it is the output gradient of convT t-1, whose bias
            # gradient (its sum over pixels) comes out of the same kernel's epilogue
            if t > 0:
                g_hi, db = conv_down(g_hi, packed[t], None, acts[t], B, H, H, CH, nchw, ACT_NONE, want_colsum=True,
                                     mask_bits=bits[t - 1])
            else:
                g_hi = conv_down(g_hi, packed[t], None, acts[t], B, H, H, CH, nchw, ACT_NONE)
        g3 = flat_transpose(g_hi.view(B, FLAT), B, to_nhwc=False)                  # grad of lin3 pre-activation
        dlw3, dlb3 = lane.run(lambda: linear_wgrad(g3, h2), g3, h2)
        g2 = linear_dgrad(g3, lins[2][0], h2, ACT_RELU, packed=lpk[2])
        dlw2, dlb2 = lane.run(lambda: linear_wgrad(g2, h1), g2, h1)
        g1 = linear_dgrad(g2, lins[1][0], h1, ACT_RELU, packed=lpk[1])
        dlw1, dlb1 = lane.run(lambda: linear_wgrad(g1, z), g1, z)
        dz = linear_dgrad(g1, lins[0][0], None, ACT_NONE, packed=lpk[0]) if ctx.needs_input_grad[0] else None
        lane.join()
        return (dz, None, None, dlw1, dlb1, dlw2, dlb2, dlw3, dlb3, *convT_grads)


# ---------------------------------------------------------------------------------------
# FactorVAE discriminator (disvae/models/discriminator.py:60-70) as ONE autograd node
# ---------------------------------------------------------------------------------------
_mlp_note_parts = 1                # trace notes of MlpFn.forward: the batch is `parts` equal row blocks noted one after the other
_mlp_skip_param_grads = False      # MlpFn.backward: input gradient only


@contextlib.contextmanager
def mlp_note_parts(parts):
    """The discriminator of FactorVAE sees both halves of the batch in ONE call; the ReLU-branch trace (start_trace) still
    lists them as the two calls the reference makes (losses.py:262,286)."""
    global _mlp_note_parts
    old, _mlp_note_parts = _mlp_note_parts, parts
    try:
        yield
    finally:
        _mlp_note_parts = old


@contextlib.contextmanager
def mlp_input_grad_only():
    """Backward passes under this context skip the weight/bias gradients of MlpFn nodes (FactorVAE: the discriminator's
    parameter gradients produced by vae_loss.backward() are zeroed before they are ever read, losses.py:277,296)."""
    global _mlp_skip_param_grads
    old, _mlp_skip_param_grads = _mlp_skip_param_grads, True
    try:
        yield
    finally:
        _mlp_skip_param_grads = old


class MlpFn(Function):
    """x -> lin(act(...)): LeakyReLU(slope) after every layer but the last."""

    @staticmethod
    def forward(ctx, x, slope, *params):
        N.require_cuda_f32(x, *params)
        x = _c(x)
        params = [_c(p) for p in params]
        n = len(params) // 2
        hs = [x]
        h = x
        lpk = linear_pack_multi([params[2 * i] for i in range(n)])
        for i in range(n):
            h = linear_fwd(h, params[2 * i], params[2 * i + 1], ACT_LEAKY if i < n - 1 else ACT_NONE, slope, packed=lpk[i])
            hs.append(h)
        if _trace is not None:
            rows = x.shape[0] // _mlp_note_parts
            for part in range(_mlp_note_parts):
                for i in range(n - 1):
                    _note("mlp.lin%d" % (i + 1), hs[i + 1][part * rows:(part + 1) * rows])
        ctx.slope, ctx.n = slope, n
        ctx.save_for_backward(*hs[:-1], *params, *lpk)
        return h

    @staticmethod
    def backward(ctx, g_out):
        n, slope = ctx.n, ctx.slope
        saved = ctx.saved_tensors
        hs, params, lpk = saved[:n], saved[n:3 * n], saved[3 * n:]
        g = _c(g_out)
        grads = [None] * (2 * n)
        dx = None
        lane = _WgradLane(g.device)
        for i in range(n - 1, -1, -1):
            if not _mlp_skip_param_grads:
                grads[2 * i], grads[2 * i + 1] = lane.run(lambda gg=g, h=hs[i]: linear_wgrad(gg, h), g, hs[i])
            if i > 0:
                g = linear_dgrad(g, params[2 * i], hs[i], ACT_LEAKY, slope, packed=lpk[i])
            elif ctx.needs_input_grad[0]:
                dx = linear_dgrad(g, params[0], None, ACT_NONE, packed=lpk[0])
        lane.join()
        return (dx, None, *grads)


# ---------------------------------------------------------------------------------------
# reparameterisation (disvae/models/vae.py:65-68)
# ---------------------------------------------------------------------------------------
def _mu_logvar(mu, logvar):
    """-> (mu, logvar, ld, row_stride) as the C ABI takes them.  [B,D] views with identical strides (the two halves of
    the encoder output) are passed as they are; anything else is made contiguous first."""
    if mu.dim() != 2 or mu.stride() != logvar.stride():
        mu, logvar = mu.contiguous(), logvar.contiguous()
        if mu.dim() != 2 or mu.stride() != logvar.stride():
            raise ValueError("mu and logvar must be [B, D] tensors of one shape, got %s and %s"
                             % (tuple(mu.shape), tuple(logvar.shape)))
    return mu, logvar, mu.stride(1), mu.stride(0)


class ReparamFn(Function):
    @staticmethod
    def forward(ctx, mu, logvar, eps, seed, offset_dev):
        N.require_cuda_f32(mu, logvar, eps)
        mu, logvar, ld, rs = _mu_logvar(mu, logvar)
        B, D = mu.shape
        z = _new((B, D), mu)
        if eps is not None:
            eps = _c(eps)
            call("dv_reparam_fwd", ptr(mu), ptr(logvar), ld, rs, ptr(eps), 0, None, ptr(z), None, B, D, stream())
        else:
            eps = _new((B, D), mu)
            call("dv_reparam_fwd", ptr(mu), ptr(logvar), ld, rs, None, seed, ptr(offset_dev), ptr(z), ptr(eps),
                 B, D, stream())
        ctx.st = (ld, rs)
        ctx.save_for_backward(logvar, eps)
        return z

    @staticmethod
    def backward(ctx, g_z):
        logvar, eps = ctx.saved_tensors
        B, D = eps.shape
        g_z = _c(g_z)
        g_mu, g_lv = torch.empty_like(eps), torch.empty_like(eps)
        call("dv_reparam_bwd", ptr(g_z), ptr(logvar), ctx.st[0], ctx.st[1], ptr(eps), ptr(g_mu), ptr(g_lv), B, D, stream())
        return g_mu, g_lv, None, None, None


# ---------------------------------------------------------------------------------------
# fused reconstruction loss + KL (losses.py:394-449, 452-480)
# ---------------------------------------------------------------------------------------
class VaeLossFn(Function):
    """-> out[2 + D] = (recon_loss, kl_total, kl_dim_0 .. kl_dim_{D-1}).
    Only out[0] and out[1] carry gradient; out[2:] are logging values (kl_loss_<i>)."""

    @staticmethod
    def forward(ctx, recon, data, mu, logvar, dist):
        N.require_cuda_f32(recon, data, mu, logvar)
        recon, data = _c(recon), _c(data)
        mu, logvar, ld, rs = _mu_logvar(mu, logvar)
        B, D = mu.shape
        n_img = recon.numel() // B
        ws = _zero_ws("vae_loss", N.lib().dv_vae_loss_workspace_bytes(B, n_img), recon.device)
        out = _new((2 + D,), recon)
        call("dv_vae_loss_fwd", ptr(recon), ptr(data), n_img, B, dist, ptr(mu), ptr(logvar), ld, rs, D,
             ptr(out), ptr(ws), stream())
        ctx.meta = (n_img, B, D, dist, ld, rs)
        ctx.save_for_backward(recon, data, mu, logvar, out)
        return out

    @staticmethod
    def backward(ctx, g_out):
        recon, data, mu, logvar, out = ctx.saved_tensors
        n_img, B, D, dist, ld, rs = ctx.meta
        g_out = _c(g_out)
        g_recon = torch.empty_like(recon) if ctx.needs_input_grad[0] else None
        g_mu = _new((B, D), mu) if ctx.needs_input_grad[2] else None
        g_lv = _new((B, D), mu) if ctx.needs_input_grad[3] else None
        call("dv_vae_loss_bwd", ptr(recon), ptr(data), n_img, B, dist, ptr(mu), ptr(logvar), ld, rs, D,
             ptr(out), ptr(g_out), ptr(g_recon), ptr(g_mu), ptr(g_lv), stream())
        return g_recon, None, g_mu, g_lv, None


# ---------------------------------------------------------------------------------------
# beta-TCVAE decomposition (losses.py:523-544 + 369-373)
# ---------------------------------------------------------------------------------------
# beta-TCVAE workspaces: the kernel leaves the header (its "last block" counter) zero, and the body carries the column
# parameters from forward to backward -- so one buffer per (B, D, device) serves every step WITHOUT a per-step zero-fill,
# as long as its previous forward has been consumed by its backward ("busy" flag; anything else gets a fresh buffer).
_bt_pool = {}


def _bt_new_workspace(B, D, device):
    """A fresh beta-TCVAE workspace: only its 16-float header must start zero (include/disvae_b200.h)."""
    ws = torch.empty((N.lib().dv_btcvae_workspace_bytes(B, D) + 3) // 4, dtype=torch.float32, device=device)
    ws[:16].zero_()
    return ws


def _bt_workspace(B, D, device):
    key = (B, D, device.index, _owner)
    ent = _bt_pool.get(key)
    if ent is not None and not ent[1]:
        ent[1] = True
        return ent[0], key
    ws = _bt_new_workspace(B, D, device)
    if ent is None:
        _bt_pool[key] = [ws, True]
        return ws, key
    return ws, None                                            # pool buffer in flight: a private one


def _btcvae_fwd(z, mu, logvar, n_data, is_mss, ws):
    """dv_btcvae_fwd over the whole batch into workspace `ws` -> (rowstats [4+D, B], terms [3])."""
    z = _c(z)
    mu, logvar, ld, rs = _mu_logvar(mu, logvar)
    B, D = z.shape
    rowstats = _new((4 + D, B), z)
    terms = _new((3,), z)
    call("dv_btcvae_fwd", ptr(z), ptr(mu), ptr(logvar), ld, rs, B, D, int(n_data), int(bool(is_mss)),
         ptr(rowstats), ptr(terms), ptr(ws), stream())
    return rowstats, terms


def _bt_release(key, ws):
    ent = _bt_pool.get(key) if key is not None else None
    if ent is not None and ent[0] is ws:
        ent[1] = False


class BtcvaeFn(Function):
    """-> terms[3] = (mi, tc, dw_kl).  ctx keeps the [4+D][B] row statistics."""

    @staticmethod
    def forward(ctx, z, mu, logvar, n_data, is_mss):
        N.require_cuda_f32(z, mu, logvar)
        B, D = z.shape
        ws, key = _bt_workspace(B, D, z.device)
        rowstats, terms = _btcvae_fwd(z, mu, logvar, n_data, is_mss, ws)
        if not (z.requires_grad or mu.requires_grad or logvar.requires_grad) or not torch.is_grad_enabled():
            _bt_release(key, ws)                               # no backward will come for it
            key = None
        ctx.meta = (B, D, int(n_data), int(bool(is_mss)), key)
        ctx.save_for_backward(rowstats, ws)
        return terms

    @staticmethod
    def backward(ctx, g_terms):
        rowstats, ws = ctx.saved_tensors
        B, D, n_data, is_mss, key = ctx.meta
        g_terms = _c(g_terms)
        g_z = _new((B, D), rowstats) if ctx.needs_input_grad[0] else None
        g_mu = _new((B, D), rowstats) if ctx.needs_input_grad[1] else None
        g_lv = _new((B, D), rowstats) if ctx.needs_input_grad[2] else None
        call("dv_btcvae_bwd", B, D, n_data, is_mss, ptr(rowstats), ptr(ws), ptr(g_terms), ptr(g_z), ptr(g_mu),
             ptr(g_lv), stream())
        _bt_release(key, ws)
        return g_z, g_mu, g_lv, None, None


class BtcvaeGlobalFn(Function):
    """beta-TCVAE terms of THIS rank's rows against the batch all-gathered from every rank (SURVEY.md 8f-1):
    the B x B log-density matrix of losses.py:523-544 is that of the GLOBAL batch B = world * b, each rank evaluates its
    row block [rank*b, (rank+1)*b) with dv_btcvae_fwd_rows, and -> terms[3] = means over its rows, so the mean of the
    ranks' terms is exactly the single-process value (equal shards).  Backward: the row side (g_z) is local and
    complete; the column side (g_mu, g_logvar) is a [B, D] partial sum over this rank's rows -> reduce-scatter.
    One all-gather of [b, 3D] forward, one reduce-scatter of [B, 2D] backward."""

    @staticmethod
    def forward(ctx, z, mu, logvar, n_data, is_mss, group):
        from . import parallel
        N.require_cuda_f32(z, mu, logvar)
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        b, D = z.shape
        B = b * world
        gathered = parallel.all_gather_rows(torch.cat([z, mu, logvar], dim=1), group)       # [B, 3D]
        zg = gathered[:, :D].contiguous()
        mug, lvg = gathered[:, D:2 * D], gathered[:, 2 * D:]                                 # ld 1, row stride 3D
        ws = _bt_new_workspace(B, D, z.device)
        rowstats = _new((4 + D, B), z)
        terms = _new((3,), z)
        call("dv_btcvae_fwd_rows", ptr(zg), ptr(mug), ptr(lvg), 1, 3 * D, B, D, rank * b, b, int(n_data), int(bool(is_mss)),
             ptr(rowstats), ptr(terms), ptr(ws), stream())
        ctx.meta = (B, D, b, rank, int(n_data), int(bool(is_mss)), group)
        ctx.save_for_backward(rowstats, ws)
        return terms

    @staticmethod
    def backward(ctx, g_terms):
        from . import parallel
        rowstats, ws = ctx.saved_tensors
        B, D, b, rank, n_data, is_mss, group = ctx.meta
        g_terms = _c(g_terms)
        g_z = _new((b, D), rowstats)
        g_cols = _new((2, B, D), rowstats)
        call("dv_btcvae_bwd_rows", B, D, rank * b, b, n_data, is_mss, ptr(rowstats), ptr(ws), ptr(g_terms), ptr(g_z),
             ptr(g_cols[0]), ptr(g_cols[1]), stream())
        mine = parallel.reduce_scatter_rows(torch.cat([g_cols[0], g_cols[1]], dim=1), group)   # [b, 2D]
        return g_z, mine[:, :D].contiguous(), mine[:, D:].contiguous(), None, None, None


def btcvae_terms(z, mu, logvar, n_data, is_mss):
    """BtcvaeFn on the weight-gradient side stream.  autograd runs a node's backward on the stream that was current when
    the node was created and synchronises producers and consumers itself, so dv_btcvae_bwd -- whose results are not
    needed before the ENCODER's backward -- overlaps with the decoder's backward pass instead of preceding it."""
    lane = _WgradLane(z.device)
    if not lane.enabled:
        return BtcvaeFn.apply(z, mu, logvar, n_data, is_mss)
    lane.side.wait_stream(lane.main)
    with torch.cuda.stream(lane.side):
        terms = BtcvaeFn.apply(z, mu, logvar, n_data, is_mss)
    lane.main.wait_stream(lane.side)
    return terms


class LossCombineFn(Function):
    """loss = sum_i coef_a[i]*a[i] + sum_j coef_b[j]*b[j] with a = the fused loss kernel's output (rec, kl, per-dim kl..:
    only the first len(coef_a) entries are weighted) and b = a short vector or 0-dim tensor (beta-TCVAE terms, the
    FactorVAE tc) or None.  One launch forward, one backward (writes the FULL gradient of `a`, zeros included) -- instead
    of the scalar select/mul/add kernels of `rec + (alpha*mi + beta*tc + ...)` and their zero-filled backward buffers."""

    @staticmethod
    def forward(ctx, a, b, coef_a, coef_b):
        import ctypes
        N.require_cuda_f32(a, b)
        a = _c(a)
        b = _c(b) if b is not None else None
        na, nb = len(coef_a), (len(coef_b) if b is not None else 0)
        ca = (ctypes.c_float * max(na, 1))(*coef_a)
        cb = (ctypes.c_float * max(nb, 1))(*(coef_b if nb else [0.0]))
        loss = _new((), a)
        call("dv_loss_combine_fwd", ptr(a), ca, na, ptr(b), cb, nb, ptr(loss), stream())
        ctx.meta = (ca, cb, na, nb, a.numel(), tuple(b.shape) if b is not None else None)
        return loss

    @staticmethod
    def backward(ctx, g):
        ca, cb, na, nb, na_total, b_shape = ctx.meta
        g = _c(g)
        g_a = _new((na_total,), g)
        g_b = _new(b_shape, g) if nb else None
        call("dv_loss_combine_bwd", ptr(g), ca, na, na_total, cb, nb, ptr(g_a), ptr(g_b), stream())
        return g_a, g_b, None, None


def _log_arg(log):
    import ctypes
    return ctypes.byref(log) if log is not None else None


class LossCombineSchedFn(Function):
    """LossCombineFn whose coefficients are formed on the device, so that a captured CUDA graph anneals: coefficient k is
    float(base[k] * linear_annealing(init, fin, step, steps_anneal)) when bit k of `sched_mask` is set (k counts coef_a,
    then coef_b), float(base[k]) otherwise.  On a training step the kernel first advances the int64 device counter `step`
    and anneals with the new value; otherwise `step` is not read (None allowed) and the annealing value is `fin`.
    `log` (a _native.LossLog, or None): the device loss log written by the same launch on a recording step.
    -> (loss, coefs): coefs [na + nb] are the float coefficients the kernel used (not differentiable)."""

    @staticmethod
    def forward(ctx, a, b, coef_a, coef_b, sched_mask, anneal, is_train, step, log):
        import ctypes
        N.require_cuda_f32(a, b)
        a = _c(a)
        b = _c(b) if b is not None else None
        na, nb = len(coef_a), (len(coef_b) if b is not None else 0)
        base = (ctypes.c_double * (na + nb))(*(list(coef_a) + (list(coef_b) if nb else [])))
        init, fin, steps_anneal = anneal
        loss, coefs = _new((), a), _new((na + nb,), a)
        call("dv_loss_combine_sched_fwd", ptr(a), na, ptr(b), nb, base, int(sched_mask), float(init), float(fin),
             int(steps_anneal), int(bool(is_train)), ptr(step), ptr(loss), ptr(coefs), _log_arg(log), stream())
        ctx.meta = (na, nb, a.numel(), tuple(b.shape) if b is not None else None)
        ctx.save_for_backward(coefs)
        ctx.mark_non_differentiable(coefs)
        return loss, coefs

    @staticmethod
    def backward(ctx, g, _g_coefs):
        coefs, = ctx.saved_tensors
        na, nb, na_total, b_shape = ctx.meta
        g = _c(g)
        g_a = _new((na_total,), g)
        g_b = _new(b_shape, g) if nb else None
        call("dv_loss_combine_sched_bwd", ptr(g), ptr(coefs), na, na_total, nb, ptr(g_a), ptr(g_b), stream())
        return g_a, g_b, None, None, None, None, None, None, None


class BetaBLossFn(Function):
    """beta-VAE_B's rec + gamma * |kl - C| (losses.py:199-200) from the fused loss kernel's output `out` = (rec, kl, ..),
    with C = linear_annealing(c_init, c_fin, step, steps_anneal) formed on the device like LossCombineSchedFn's
    coefficients (C_fin outside training).  Forward and backward are bit-identical to that torch expression and its
    autograd gradient.  -> (loss, consts): consts = (C, gamma) as floats (not differentiable)."""

    @staticmethod
    def forward(ctx, out, gamma, c_anneal, is_train, step, log):
        N.require_cuda_f32(out)
        out = _c(out)
        c_init, c_fin, steps_anneal = c_anneal
        loss, consts = _new((), out), _new((2,), out)
        call("dv_betab_loss_fwd", ptr(out), float(gamma), float(c_init), float(c_fin), int(steps_anneal),
             int(bool(is_train)), ptr(step), ptr(loss), ptr(consts), _log_arg(log), stream())
        ctx.save_for_backward(out, consts)
        ctx.mark_non_differentiable(consts)
        return loss, consts

    @staticmethod
    def backward(ctx, g, _g_consts):
        out, consts = ctx.saved_tensors
        g = _c(g)
        g_out = torch.empty_like(out)
        call("dv_betab_loss_bwd", ptr(g), ptr(out), ptr(consts), out.numel(), ptr(g_out), stream())
        return g_out, None, None, None, None, None


def loss_record(step, log):
    """The device loss log on its own (dv_loss_record), predicated on the counter `step` as it stands."""
    call("dv_loss_record", ptr(step), _log_arg(log), stream())


def btcvae_rowstats(z, mu, logvar, n_data, is_mss=True):
    """(log_pz, log_qz, log_prod_qzi, log_q_zCx) like losses.py:523-544 (no autograd)."""
    with torch.no_grad():
        B, D = z.shape
        rowstats, _ = _btcvae_fwd(z, mu, logvar, n_data, is_mss, _bt_new_workspace(B, D, z.device))
    return rowstats[0], rowstats[1], rowstats[2], rowstats[3]


# ---------------------------------------------------------------------------------------
# FactorVAE heads (losses.py:265, 291-295, 483-508)
# ---------------------------------------------------------------------------------------
_PERM_MAX_B = 4096      # dv_permute_dims generates device permutations of at most this many rows


def permute_dims(z, perms=None, seed=0, offset_dev=None):
    N.require_cuda_f32(z)
    z = _c(z.detach())
    B, D = z.shape
    if perms is None and B > _PERM_MAX_B:
        return permute_dims_rows(z, 0, B, None, seed, offset_dev)
    out = torch.empty_like(z)
    if perms is not None:
        perms = perms.to(device=z.device, dtype=torch.int64).contiguous()
        call("dv_permute_dims", ptr(z), ptr(perms), 0, None, ptr(out), B, D, stream())
    else:
        call("dv_permute_dims", ptr(z), None, seed, ptr(offset_dev), ptr(out), B, D, stream())
    return out


def permute_dims_rows(z, row0, nrows, perms=None, seed=0, offset_dev=None):
    """Rows [row0, row0 + nrows) of permute_dims(z, perms, seed, offset_dev), at any batch size: the permutation is
    the one of all B rows of z, and the device offset advances by B*D whatever the window."""
    N.require_cuda_f32(z)
    z = _c(z.detach())
    B, D = z.shape
    out = torch.empty((nrows, D), dtype=torch.float32, device=z.device)
    if perms is not None:
        perms = perms.to(device=z.device, dtype=torch.int64).contiguous()
        call("dv_permute_dims_rows", ptr(z), ptr(perms), 0, None, ptr(out), B, D, row0, nrows, None, stream())
    else:
        nbytes = N.lib().dv_permute_dims_workspace_bytes(B, D)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=z.device) if nbytes else None
        call("dv_permute_dims_rows", ptr(z), None, seed, ptr(offset_dev), ptr(out), B, D, row0, nrows, ptr(ws), stream())
    return out


class FactorTcFn(Function):
    @staticmethod
    def forward(ctx, d_z):
        N.require_cuda_f32(d_z)
        d_z = _c(d_z)
        tc = _new((), d_z)
        call("dv_factor_tc_fwd", ptr(d_z), d_z.shape[0], ptr(tc), stream())
        ctx.h = d_z.shape[0]
        return tc

    @staticmethod
    def backward(ctx, g):
        g = _c(g)
        out = torch.empty((ctx.h, 2), dtype=torch.float32, device=g.device)
        call("dv_factor_tc_bwd", ptr(g), ctx.h, ptr(out), stream())
        return out


class FactorCeFn(Function):
    @staticmethod
    def forward(ctx, d_z, d_perm):
        N.require_cuda_f32(d_z, d_perm)
        d_z, d_perm = _c(d_z), _c(d_perm)
        out = _new((), d_z)
        call("dv_factor_ce_fwd", ptr(d_z), ptr(d_perm), d_z.shape[0], ptr(out), stream())
        ctx.save_for_backward(d_z, d_perm)
        return out

    @staticmethod
    def backward(ctx, g):
        d_z, d_perm = ctx.saved_tensors
        g = _c(g)
        g_z, g_p = torch.empty_like(d_z), torch.empty_like(d_perm)
        call("dv_factor_ce_bwd", ptr(d_z), ptr(d_perm), ptr(g), d_z.shape[0], ptr(g_z), ptr(g_p), stream())
        return g_z, g_p


def adam_step(param_flat, grad_flat, exp_avg, exp_avg_sq, step_dev, lr, betas, eps, grad_scale=1.0):
    call("dv_adam_step", ptr(param_flat), ptr(grad_flat), ptr(exp_avg), ptr(exp_avg_sq), ptr(step_dev),
         param_flat.numel(), lr, betas[0], betas[1], eps, grad_scale, stream())
