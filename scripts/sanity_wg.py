"""wgrad32 kernel check: accuracy against an fp64 reference over the geometries of the networks (and ragged batches),
then timing at the bench shapes.  Exit 1 = accuracy, anything else non-zero = crash / hang (run under `timeout`)."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))
from disvae import ops
torch.manual_seed(0)
d = torch.device("cuda")
nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
worst = 0.0
for (B, H) in ((3, 4), (37, 4), (64, 8), (33, 8), (170, 16), (1024, 4), (600, 16)):
    hi = torch.randn(B, 32, 2 * H, 2 * H)
    lo = torch.randn(B, 32, H, H)
    dw, db = ops.conv_wgrad(nhwc(lo).to(d), nhwc(hi).to(d), B, H, H, 32, 0, True)
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(hi.double(), (32, 32, 4, 4), lo.double(), stride=2, padding=1)
    e = ((dw.cpu().double() - ref).abs().max() / ref.abs().max()).item()
    eb = ((db.cpu().double() - lo.double().sum((0, 2, 3))).abs().max() / lo.double().sum((0, 2, 3)).abs().max()).item()
    print("sanity_wg: B=%d H=%d  dw err %.2e  db err %.2e" % (B, H, e, eb), flush=True)
    worst = max(worst, e, eb)
for (Bt, H) in ((1024, 16), (1024, 8), (1024, 4)):
    xt = torch.randn(Bt, 2 * H, 2 * H, 32, device=d); lt = torch.randn(Bt, H, H, 32, device=d)
    fn = lambda: ops.conv_wgrad(lt, xt, Bt, H, H, 32, 0, True)
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        fn()
    e1.record(); torch.cuda.synchronize()
    print("sanity_wg timing: B=%d H=%d %.1f us (kernel + split-K reduce)" % (Bt, H, e0.elapsed_time(e1) / 20 * 1e3), flush=True)
sys.exit(0 if worst < 4e-6 else 1)
