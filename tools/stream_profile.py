"""per-op device time of ONE streaming step (config 5: dagr-l, 640x480, 1 ms chunks of a 1 Mevents/s stream, 50 ms window):
the step is run eagerly with CUDA events around every C-ABI call (the production path replays it as one CUDA graph)."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import StreamingDetector, pack_stage, synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H = 640, 480
size = sys.argv[1] if len(sys.argv) > 1 else "l"
torch.manual_seed(0)
model = randomize_bn(DAGR(default_args(size, batch_size=1), height=H, width=W).eval()).cuda()
x, y, t, p = synth_stream(1_000_000, 0.2, W, H)
det = StreamingDetector(model, window_us=50_000, max_chunk=4096)
bounds = np.searchsorted(t, np.arange(0, 200_001, 1000))
for k in range(80):
    a, b = int(bounds[k]), int(bounds[k + 1])
    det.push(x[a:b], y[a:b], t[a:b], p[a:b], (k + 1) * 1000)
torch.cuda.synchronize()
eng = model.engine
eng.prof = {}
for k in range(80, 110):
    a, b = int(bounds[k]), int(bounds[k + 1])
    pack_stage(det._stage_np, [(x[a:b], y[a:b], t[a:b], p[a:b])], [(k + 1) * 1000 - det.window_us], det.max_chunk)
    det._enqueue()
torch.cuda.synchronize()
prof = eng.prof_summary()
eng.prof = None
rows = sorted(((v["ms"] * v["calls"] / 30, k, v["calls"] // 30, v["ms"]) for k, v in prof.items()), reverse=True)
print(json.dumps(dict(model=f"dagr-{size}", total_ms_per_step=sum(r[0] for r in rows),
                      per_op=[dict(op=k, calls_per_step=c, ms_each=round(m, 4), ms_per_step=round(tot, 4)) for tot, k, c, m in rows])))
