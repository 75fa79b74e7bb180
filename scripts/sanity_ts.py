"""Quick guard before a long GPU run: the tensor-core 32->32 conv kernels must complete and be fp32-grade accurate
(SANITY_TIME=1 also times them at the bench shape).  Run under `timeout`: a hang here must not eat the test budget."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))
from disvae import ops
import torch.nn.functional as F
torch.manual_seed(0)
B, H = 300, 16
x = torch.randn(B, 32, 2 * H, 2 * H)
lo = torch.randn(B, 32, H, H)
w = torch.randn(32, 32, 4, 4) * 0.1
d = torch.device("cuda")
wp = ops.conv_pack(w.to(d), 32)
nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
which = sys.argv[1] if len(sys.argv) > 1 else "both"
B = int(os.environ.get("SANITY_B", B))
x, lo = x[:B], lo[:B]
got_d = ops.conv_down(nhwc(x).to(d), wp, None, None, B, H, H, 32, 0, 1) if which != "up" else None
torch.cuda.synchronize()
got_u = ops.conv_up(nhwc(lo).to(d), wp, None, None, B, H, H, 32, 0, 1) if which != "down" else None
torch.cuda.synchronize()
if which != "both":
    print("sanity_ts: %s completed" % which)
    sys.exit(0)
if os.environ.get("SANITY_TIME") == "1":          # timing of both kernels at the bench shapes (B = 1024)
    Bt = 1024
    for Ht in (16, 8, 4):
        xt = torch.randn(Bt, 2 * Ht, 2 * Ht, 32, device=d); lt = torch.randn(Bt, Ht, Ht, 32, device=d)
        mlo = torch.randn(Bt, Ht, Ht, 32, device=d); mhi = torch.randn(Bt, 2 * Ht, 2 * Ht, 32, device=d)
        words = lambda t: torch.where((w := ((t > 0).long() << torch.arange(32, device=d)).sum(-1)) >= 2 ** 31, w - 2 ** 32, w).int()
        blo, bhi = words(mlo), words(mhi)
        for name, fn in (("down", lambda: ops.conv_down(xt, wp, None, None, Bt, Ht, Ht, 32, 0, 1)),
                         ("down+bits_out", lambda: ops.conv_down(xt, wp, None, None, Bt, Ht, Ht, 32, 0, 1, want_bits=True)),
                         ("down+mask", lambda: ops.conv_down(xt, wp, None, mlo, Bt, Ht, Ht, 32, 0, 0)),
                         ("down+mask_bits", lambda: ops.conv_down(xt, wp, None, mlo, Bt, Ht, Ht, 32, 0, 0, mask_bits=blo)),
                         ("up", lambda: ops.conv_up(lt, wp, None, None, Bt, Ht, Ht, 32, 0, 1)),
                         ("up+bits_out", lambda: ops.conv_up(lt, wp, None, None, Bt, Ht, Ht, 32, 0, 1, want_bits=True)),
                         ("up+mask", lambda: ops.conv_up(lt, wp, None, mhi, Bt, Ht, Ht, 32, 0, 0)),
                         ("up+mask_bits", lambda: ops.conv_up(lt, wp, None, mhi, Bt, Ht, Ht, 32, 0, 0, mask_bits=bhi))):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                fn()
            e1.record(); torch.cuda.synchronize()
            print("sanity_ts timing: H=%d %s %.1f us" % (Ht, name, e0.elapsed_time(e1) / 20 * 1e3), flush=True)
ref_d = torch.relu(F.conv2d(x.double(), w.double(), None, stride=2, padding=1))
ref_u = torch.relu(F.conv_transpose2d(lo.double(), w.double(), None, stride=2, padding=1))
ed = ((got_d.cpu().permute(0, 3, 1, 2).double() - ref_d).abs().max() / ref_d.abs().max()).item()
eu = ((got_u.cpu().permute(0, 3, 1, 2).double() - ref_u).abs().max() / ref_u.abs().max()).item()
print("sanity_ts: down err %.2e up err %.2e" % (ed, eu))
sys.exit(0 if ed < 1e-5 and eu < 1e-5 else 1)
