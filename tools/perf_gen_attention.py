"""Speed of the generalized attention blocks on the GPU: whole R-50 steps with and without the published c4-c5 layout, every
attention launch of that layout alone, and a torch restatement of the reference's materialised formulation for context.

    python tools/perf_gen_attention.py [--batch 16] [--reps 5] [--out perf_gen_attention.json]

Step times: 16 tiles of 1024^2, the dense graph (backbone + FPN + head) captured as one CUDA graph per model, models
alternating, median of `reps` rounds of 10 replays.  Launch times: CUDA events over 50 launches after 5 warm-up launches.
Algorithmic FLOPs of a launch: 2 N HW HkWk C for Q.K, the same for P.V, and 2 N HW (Hk + Wk) C for the position rows; the f16x3
rate counts three MMAs per product.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orientedreppoints_b200 import gen_attention as ga                              # noqa: E402
from orientedreppoints_b200.detector import OrientedRepPointsDetector               # noqa: E402
from orientedreppoints_b200.weights import gen_attention_layout, gen_attention_spec, random_state_dict   # noqa: E402

PUB = dict(spatial_range=-1, num_heads=8, kv_stride=2)
STAGES = [[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]]
PEAK = 989.0                                            # H100 SXM data sheet, dense fp16 / bf16 TFLOP/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def detector(t, fmt, dev):
    kw = {} if t is None else dict(gen_attention=dict(PUB, attention_type=t), stage_with_gen_attention=STAGES)
    sd = random_state_dict(50, seed=0, **kw)
    lay = None if t is None else gen_attention_layout(50, dict(PUB, attention_type=t), STAGES)
    return OrientedRepPointsDetector(sd, 50, dev, fmt, gen_attention=lay)


def step_times(fmt, batch, reps, dev):
    img = torch.randn(batch, 3, 1024, 1024, device=dev)
    dets = {name: detector(t, fmt, dev).capture(tuple(img.shape)) for name, t in (("R-50", None), ("R-50 + 0010", "0010"),
                                                                                   ("R-50 + 1111", "1111"))}
    times = {k: [] for k in dets}
    for _ in range(reps):
        for name, d in dets.items():                                   # models alternate
            d.forward_dense_graph(img)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(10):
                d.forward_dense_graph(img)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / 10)
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


def launch_times(fmt, batch, dev):
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    e = EngineTCSplit(dev) if fmt == "f16x3" else EngineTC(dev)
    out = []
    for t in ("1111", "0010"):
        for li, (h, c) in ((2, (64, 256)), (3, (32, 512))):
            cfg = dict(PUB, attention_type=t)
            stages = [[], [], [], []]
            stages[li] = [0]
            sd = random_state_dict(50, seed=1, gen_attention=cfg, stage_with_gen_attention=stages)
            blk = ga.GenAttentionBlock(sd, "backbone.layer%d.0" % (li + 1), gen_attention_spec(cfg, c), dev)
            x = e.from_float(torch.randn(batch, h, h, c, device=dev))
            kv = e.conv(x, blk.kv)
            hk = -(-h // 2)
            if blk.saliency:
                q, qh = blk.bias_rows(e, batch), 1
                args = (q, 0, None, kv, blk.k_off, blk.v_off, None, batch, 1, 1, hk, hk, 2, c, 8)
            else:
                q, qh = e.conv(x, blk.q), h
                args = (q, blk.qc_off, blk.qp_off, kv, blk.k_off, blk.v_off, blk.tables(e, h, h), batch, h, h, hk, hk, 2, c, 8)
            for _ in range(5):
                ga.attend(e, *args)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(50):
                ga.attend(e, *args)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / 50
            hw, nk = qh * qh, hk * hk
            flops = 4.0 * batch * hw * nk * c + (2.0 * batch * hw * 2 * hk * c if blk.qp_off is not None else 0.0)
            tf = flops / ms / 1e9 * (3 if fmt == "f16x3" else 1)
            out.append(dict(type=t, stage="c%d" % (li + 2), map=h, keys=nk, channels=c, us=round(ms * 1e3, 1),
                            algorithmic_tflops=round(tf, 1), share_of_peak=round(tf / PEAK, 3)))
    return out


def materialised(dev, n=2):
    """the reference's formulation in torch (fp32, stage c4 at 1024^2, '1111'): the [n, 8, 4096, 1024] energy written out"""
    h, c, heads, d = 64, 256, 8, 32
    q = torch.randn(n, heads, h * h, d, device=dev)
    k = torch.randn(n, heads, d, 1024, device=dev)
    v = torch.randn(n, heads, 1024, d, device=dev)
    px = torch.randn(n, heads, h, 32, d, device=dev)
    py = torch.randn(n, heads, h, 32, d, device=dev)

    def run():
        e = torch.matmul(q, k).view(n, heads, h, h, 32, 32)
        q5 = q.view(n, heads, h, h, d)
        ex = torch.matmul(q5.permute(0, 1, 3, 2, 4), px.permute(0, 1, 2, 4, 3)).permute(0, 1, 3, 2, 4).unsqueeze(4)
        ey = torch.matmul(q5, py.permute(0, 1, 2, 4, 3)).unsqueeze(5)
        e = (e + ex + ey).view(n, heads, h * h, 1024)
        return torch.matmul(torch.softmax(e, 3), v)

    for _ in range(3):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        run()
    b.record()
    torch.cuda.synchronize()
    return dict(batch=n, stage="c4", map=h, ms=round(a.elapsed_time(b) / 10, 3), energy_bytes=n * heads * h * h * 1024 * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_gen_attention needs a GPU: there is no CPU measurement")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(card=card(), batch=a.batch, tile=1024)
    for fmt in ("f16x3", "bf16"):
        res[fmt] = dict(step_ms=step_times(fmt, a.batch, a.reps, dev), launches=launch_times(fmt, a.batch, dev))
    res["torch_materialised_fp32"] = materialised(dev)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
