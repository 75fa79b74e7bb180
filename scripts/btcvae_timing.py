"""Phase boundaries of the single-launch beta-TCVAE forward kernel (block 0, SM clocks) warm and after an L2 flush.
DV_BTCVAE_TIMING=1."""
import os, sys, torch
os.environ["DV_BTCVAE_TIMING"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))
from disvae import _native as N
from disvae._native import ptr, stream
dev = torch.device("cuda", 0)
B, D = 1024, 10
torch.manual_seed(1)
mu = torch.randn(B, D, device=dev); lv = torch.randn(B, D, device=dev) * 0.5 - 1
z = mu + torch.exp(0.5 * lv) * torch.randn(B, D, device=dev)
L = N.lib()
ws = torch.zeros((L.dv_btcvae_workspace_bytes(B, D) + 3) // 4, device=dev)
rs = torch.empty(4 + D, B, device=dev); terms = torch.empty(3, device=dev)
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
def run(cold):
    if cold:
        flush.fill_(1.0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    N.call("dv_btcvae_fwd", ptr(z), ptr(mu), ptr(lv), 1, D, B, D, 737280, 1, ptr(rs), ptr(terms), ptr(ws), stream())
    e1.record(); torch.cuda.synchronize()
    off = 16 + 4 * B * D + 4 * 128 + 16                   # header | pj[D][B] float4 | blockpart[128 blocks][4] | 16 floats
    marks = ws[off:off + 6].tolist()
    timers = ws[off + 16:off + 16 + 4 * 128].view(torch.int64).view(128, 2).cpu()
    return e0.elapsed_time(e1) * 1e3, marks, timers
for i in range(5): run(False)
for cold in (False, True):
    rows = [run(cold) for _ in range(9)]
    rows.sort(key=lambda r: r[0])
    us, marks, timers = rows[len(rows) // 2]
    t0 = timers[:, 0].min().item()
    st, en = (timers[:, 0] - t0).float() / 1e3, (timers[:, 1] - t0).float() / 1e3
    print("   per-block global timer (us since the first block's entry): entry min/median/max %.2f %.2f %.2f | exit min/median/max %.2f %.2f %.2f"
          % (st.min(), st.median(), st.max(), en.min(), en.median(), en.max()))
    names = "(unused) | stage+fold | sweep | cluster.sync | finalise | exit sync"
    print("cold" if cold else "warm", "event us %.2f" % us, "marks (clk since entry): %s =" % names, [int(m) for m in marks],
          " => us @1.9GHz:", [round(m / 1900, 2) for m in marks])
