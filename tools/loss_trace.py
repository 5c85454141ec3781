"""Scratch probe (measurement build with -DOM_LOSS_TRACE): per-CTA event times of the gradient GEMMs."""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200 import _lib as om_lib  # noqa: E402

lib = om_lib.load()
raw = ctypes.CDLL(om_lib.LIB_PATH)
dev = torch.device("cuda:0")
bq, bp = 512, 4096
g = torch.Generator().manual_seed(1)
xq = (torch.randn(bq, 768, generator=g) * 0.5).to(torch.bfloat16).to(dev)
xp = (torch.randn(bp, 768, generator=g) * 0.5).to(torch.bfloat16).to(dev)
lo = torch.empty((), device=dev)
dq, dp = torch.empty(bq, 768, device=dev), torch.empty(bp, 768, device=dev)
which = os.environ.get("OM_PROBE_GRADS", "both")
for _ in range(5):
    om_lib.check(lib.om_contrastive_loss_fwd_bwd(xq.data_ptr(), xp.data_ptr(), om_lib.OM_BF16, bq, bp, 768, None,
                                                 om_lib.OM_REDUCE_MEAN, 1.0, lo.data_ptr(),
                                                 dq.data_ptr() if which != "dp" else None,
                                                 dp.data_ptr() if which != "dq" else None, None,
                                                 om_lib.current_stream_ptr()))
torch.cuda.synchronize()
ctas = min(om_lib.check(lib.om_device_sm_count()), 160)  # the loss grid is at most one CTA per SM; the trace holds 160
buf = np.zeros((ctas, 64), np.uint64)
raw.om_debug_loss_trace(buf.ctypes.data_as(ctypes.c_void_p), ctas)
t = buf.astype(np.int64)
t0 = t[:, 60].min()
rel = np.where(t >= t0, t - t0, -1)
names = ["tma0", "full0", "-", "mma_done", "stored", "fenced", "reduced", "-"]
np.set_printoptions(linewidth=250)
print("which =", which, " grads start spread (ns):", int(t[:, 60].max() - t0), " end (slot 61): min/max",
      int(rel[:, 61].min()), int(rel[:, 61].max()))
for item in range(5):
    for e in range(7):
        col = rel[:, item * 8 + e]
        ok = col[col >= 0]
        if ok.size:
            print("item %d %-8s n=%3d  min %6d  med %6d  max %6d" % (item, names[e], ok.size, ok.min(), int(np.median(ok)), ok.max()))
for c in sorted({0, 1, ctas // 3, ctas // 2, ctas - 1}):
    print("cta", c, rel[c, :48].reshape(6, 8)[:, :7].tolist(), "end", rel[c, 61])
