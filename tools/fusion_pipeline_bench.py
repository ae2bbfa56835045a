"""PipelinedDetector on image-fusion batches against model(data) per batch, on config 3's model (dagr-s + ResNet-50,
640x480, seeded random weights with randomised BN), at B = 8 and B = 1, in TF32 and bf16:
  * inputs: four pinned host batches of raw events (300 k per sample, uniform, 50 ms) and u8 frames, fed through
    Prefetcher(transform=format_data), so the H2D copy and the formatting of step i+1 overlap step i in both routes;
  * route "model": det = model(pf.next())[0], detections copied to the host (one synchronisation per batch);
  * route "pipelined": PipelinedDetector.submit(pf.next()), handle i resolved after batch i+1 was submitted;
  * five rounds, the routes alternated within each, ms per batch (host clock around a loop that ends with every
    detection on the host), the slowest batch of each round (host time from one result() to the next), whether a graph
    was captured again inside a timed round and the reserved memory after it; the detections of the two routes are
    asserted equal batch for batch;
  * device memory of one set of image-branch graphs (trunk activations + outputs) at each shape, and the growth of the
    reserved memory when the pipelined route is first used;
  * a separate torch.profiler run of the pipelined route (B = 8, TF32): per coarse stack, the time a trunk kernel ran
    beside it; how long trunk kernels ran beside event-level kernels, the share of the trunk stream's span it was busy,
    and the kernel time of all streams per step against the trace's span per step; from the kernels' streams and time stamps (the trace itself is written next to the JSON).
The card's name and power limit are read in the same call.  Writes OUT/h100_fusion_pipeline.json
(usage: python tools/fusion_pipeline_bench.py OUT)."""
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.data import format_data, synth_batch
from dagr_b200.model.dagr import DAGR
from dagr_b200.model.image_branch import branch_of
from dagr_b200.pipeline import PipelinedDetector, Prefetcher
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H, EVENTS, STEPS, WARM, ROUNDS = 640, 480, 300_000, 24, 6, 5
if len(sys.argv) != 2:
    sys.exit("usage: python tools/fusion_pipeline_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")
smi = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
card = subprocess.run(smi, capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock):", card, flush=True)


def model_s(B):
    torch.manual_seed(0)
    return randomize_bn(DAGR(default_args("s", batch_size=B, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)


def pinned(B):
    return [synth_batch(B, EVENTS, W, H, seed=4242 + 10 * i, kind="uniform", with_image=True).pin_memory() for i in range(4)]


def host(dets):
    return [(x["boxes"].cpu(), x["scores"].cpu(), x["labels"].cpu()) for x in dets]


STAMPS = []                                                       # host time at which each batch's detections arrived


def run_model(m, pf, n):
    res = []
    for _ in range(n):
        res.append(host(m(pf.next())[0]))
        STAMPS.append(time.perf_counter())
    return res


def run_pipelined(pd, pf, n):
    res, prev = [], None
    for _ in range(n):
        h = pd.submit(pf.next())
        if prev is not None:
            res.append(host(prev.result()))
            STAMPS.append(time.perf_counter())
        prev = h
    res.append(host(prev.result()))
    STAMPS.append(time.perf_counter())
    return res


def graph_ids(m):
    """identities of every captured graph of the model (coarse stacks per slot, image-branch stages): a change inside a
    timed round means a capture happened in it."""
    ids = {id(sw["graph"][1]) for ws in m.engine._ws.values() for sw in ws.get("slots", {}).values() if sw.get("graph") is not None}
    return ids | {id(st.get("g1")) for st in branch_of(m)._graphs.values() if st.get("g1") is not None}


def timed(fn, *a):
    torch.cuda.synchronize()
    STAMPS.clear()
    t0 = time.perf_counter()
    r = fn(*a, STEPS)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    gaps = [b - a for a, b in zip([t0] + STAMPS[:-1], STAMPS)]
    return (t1 - t0) * 1e3 / STEPS, round(max(gaps) * 1e3, 3), r


def same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for da, db in zip(a, b) for sa, sb in zip(da, db) for x, y in zip(sa, sb))


def branch_set_bytes(m, batches):
    """reserved device memory of one more set of image-branch graphs (stage 1 + 2 activations and outputs) at this shape."""
    img = batches[0].image.to(dev).float() / 255.0
    br = branch_of(m)
    torch.cuda.synchronize()
    r0, a0 = torch.cuda.memory_reserved(dev), torch.cuda.memory_allocated(dev)
    for _ in range(3):
        br.run(img, use_graph=True, precision=m.image_precision, slot=7)
    torch.cuda.synchronize()
    r1, a1 = torch.cuda.memory_reserved(dev), torch.cuda.memory_allocated(dev)
    key = (tuple(img.shape), str(dev), m.image_precision, 7)
    st = br._graphs.pop(key)
    outs = sum(t.numel() * t.element_size() for t in list(st["f12"]) + list(st["f345"]) + [t for v in st["outs"].values() for t in v])
    del st
    torch.cuda.synchronize()
    return dict(reserved_mb=round((r1 - r0) / 2 ** 20, 1), allocated_mb=round((a1 - a0) / 2 ** 20, 1), outputs_mb=round(outs / 2 ** 20, 1))


results = {}
for B in (8, 1):
    m = model_s(B)
    batches = pinned(B)
    pd = PipelinedDetector(m)
    # one Prefetcher per route for the whole run: the caching allocator keeps the blocks of a stream for that stream, so
    # a new Prefetcher (a new side stream) per loop would leave the previous one's blocks reserved
    pf_m, pf_p = Prefetcher(batches, dev, transform=format_data), Prefetcher(batches, dev, transform=format_data)
    for prec in ("tf32", "bf16"):
        m.image_precision = prec
        run_model(m, pf_m, WARM)
        torch.cuda.synchronize()
        r_before = torch.cuda.memory_reserved(dev)
        run_pipelined(pd, pf_p, WARM)
        torch.cuda.synchronize()
        grow = round((torch.cuda.memory_reserved(dev) - r_before) / 2 ** 20, 1)
        rec = dict(rounds=[], pipelined_first_use_reserved_growth_mb=grow, branch_graph_set=branch_set_bytes(m, batches))
        for rnd in range(ROUNDS):
            g0 = graph_ids(m)
            t_m, w_m, d_m = timed(run_model, m, pf_m)
            g1 = graph_ids(m)
            t_p, w_p, d_p = timed(run_pipelined, pd, pf_p)
            g2 = graph_ids(m)
            assert same(d_m, d_p), f"B={B} {prec} round {rnd}: the pipelined detections differ from model(data)"
            ndet = sum(x[0].shape[0] for d in d_m for x in d)
            rec["rounds"].append(dict(model_ms_per_batch=round(t_m, 3), pipelined_ms_per_batch=round(t_p, 3),
                                      model_slowest_batch_ms=w_m, pipelined_slowest_batch_ms=w_p,
                                      captured_in_round=dict(model=g1 != g0, pipelined=g2 != g1),
                                      reserved_mb_after=round(torch.cuda.memory_reserved(dev) / 2 ** 20, 1),
                                      detections=int(ndet), equal=True))
            print(f"B={B} {prec} round {rnd}: model(data) {t_m:.3f} ms/batch (slowest {w_m}), pipelined {t_p:.3f} ms/batch "
                  f"(slowest {w_p}), captures {g1 != g0}/{g2 != g1}, {ndet} detections equal", flush=True)
        med = lambda k: round(sorted(r[k] for r in rec["rounds"])[ROUNDS // 2], 3)
        ms_m, ms_p = med("model_ms_per_batch"), med("pipelined_ms_per_batch")
        rec.update(model_ms_per_batch=ms_m, pipelined_ms_per_batch=ms_p, speedup=round(ms_m / ms_p, 3),
                   rounds_pipelined_slower=sum(r["pipelined_ms_per_batch"] > r["model_ms_per_batch"] for r in rec["rounds"]))
        print(f"B={B} {prec}: memory {rec['branch_graph_set']}, pipelined first use +{grow} MB reserved", flush=True)
        results[f"batch{B}_{prec}"] = rec
    del m, pd, batches, pf_m, pf_p
    torch.cuda.empty_cache()


# ---- profiled run: does the trunk of batch i+1 run beside the coarse stack of batch i? ----------------------------------
def overlap_report(trace_path):
    ev = [e for e in json.loads(Path(trace_path).read_text())["traceEvents"] if e.get("cat") == "kernel"]
    by_stream = {}
    for e in ev:
        by_stream.setdefault(e["args"].get("stream"), []).append((e["ts"], e["ts"] + e["dur"], e["name"]))
    coarse = next(s for s, ks in by_stream.items() if any("k_postprocess_nms" in k[2] for k in ks))
    event_level = {s for s, ks in by_stream.items() if any("l1_build" in k[2] or "l1_conv" in k[2] for k in ks)}
    others = {s: ks for s, ks in by_stream.items() if s != coarse and s not in event_level
              and not any("k_grid" in k[2] or "k_head_finish" in k[2] for k in ks)}
    trunk = max(others, key=lambda s: sum(k[1] - k[0] for k in others[s]))
    tk = sorted(by_stream[trunk])
    stacks, cur = [], []
    for k in sorted(by_stream[coarse]):
        cur.append(k)
        if "k_postprocess_nms" in k[2]:
            stacks.append((cur[0][0], k[1]))
            cur = []
    def union(iv):
        out = []
        for t0, t1 in sorted(iv):
            if out and t0 <= out[-1][1]:
                out[-1][1] = max(out[-1][1], t1)
            else:
                out.append([t0, t1])
        return out
    tu = union([(t0, t1) for t0, t1, _ in tk])
    eu = union([(t0, t1) for s in event_level for t0, t1, _ in by_stream[s]])
    beside_ev = sum(max(0.0, min(b1, e1) - max(a1, e0)) for a1, b1 in tu for e0, e1 in eu)
    busy = sum(b1 - a1 for a1, b1 in tu) / max(tu[-1][1] - tu[0][0], 1e-9)
    rows = []
    for a, b in stacks:
        ov = sum(max(0.0, min(b, t1) - max(a, t0)) for t0, t1, _ in tk)
        rows.append(dict(coarse_stack_us=round(b - a, 1), trunk_kernels_beside_us=round(ov, 1)))
    return dict(streams=dict(coarse=coarse, trunk=trunk, event_level=sorted(event_level)), trunk_kernels=len(tk),
                trunk_beside_event_level_us=round(beside_ev, 1), trunk_stream_busy_share=round(busy, 4),
                kernel_us_per_step=round(sum(e["dur"] for e in ev) / len(stacks), 1),
                span_us_per_step=round((max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)) / len(stacks), 1),
                per_step=rows, steps_with_trunk_beside=sum(r["trunk_kernels_beside_us"] > 0 for r in rows))


m = model_s(8)
batches = pinned(8)
pd = PipelinedDetector(m)
pf = Prefetcher(batches, dev, transform=format_data)
run_pipelined(pd, pf, WARM)
torch.cuda.synchronize()
trace = out_dir / "fusion_pipeline_b8_tf32.pt.trace.json"
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
    run_pipelined(pd, pf, 6)
    torch.cuda.synchronize()
prof.export_chrome_trace(str(trace))
try:
    profile = overlap_report(trace)
except Exception as e:                                           # the timings above stand without the trace summary
    profile = dict(error=repr(e))
print("profile:", json.dumps(profile), flush=True)

doc = dict(
    card=card,
    workload=(f"config 3's model: dagr-s + ResNet-50 image fusion, {W}x{H}, seeded random weights with randomised BN; "
              f"{EVENTS} uniform events per sample in a 50 ms window and one u8 frame per sample, four pinned host batches "
              "through Prefetcher(transform=format_data)"),
    method=(f"per route {STEPS} batches after {WARM} warm-up batches, host clock around the loop, which ends with every detection on "
            f"the host; {ROUNDS} rounds, routes alternated; ms_per_batch fields are the median round, every round is in `rounds` "
            "(slowest batch = longest host interval between two batches' detections; captured_in_round = a graph was captured "
            "during the timed loop); detections asserted equal"),
    routes=dict(model="model(pf.next())[0] and the detections copied to the host, one batch at a time",
                pipelined="PipelinedDetector.submit(pf.next()); handle i resolved after batch i+1 was submitted"),
    memory_note=("branch_graph_set: reserved / allocated device memory of one more set of image-branch graphs at the shape (the "
                 "pipelined route keeps one per hand-off slot, two sets, beside the one model(data) uses); outputs_mb: its taps and "
                 "head maps alone.  pipelined_first_use_reserved_growth_mb: reserved memory added by the first pipelined steps "
                 "after model(data) had run (both slots' branch graphs, the engine's second hand-off slot, the coarse graphs)"),
    results=results,
    profile_b8_tf32=dict(note=("torch.profiler over 6 pipelined batches: per coarse stack (its first kernel to its NMS, on the "
                               "engine's side stream), the kernel time of the image trunk's stream inside that interval; the "
                               "coarse stack of batch i waits for batch i's whole trunk, so trunk kernels beside it belong to "
                               "later batches"), **profile),
)
(out_dir / "h100_fusion_pipeline.json").write_text(json.dumps(doc, indent=1))
print("wrote", out_dir / "h100_fusion_pipeline.json", flush=True)
