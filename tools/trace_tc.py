"""per-launch trace of the tensor-core convolutions of one dense step: every conv_tc_kernel launch of one eager pass in
launch order (shape, plan, torch.profiler kernel time), the total of the library's CUDA-event pairs around the same
launches, and the whole graph step
    python tools/trace_tc.py <tiles> [f16x3|bf16] [depth]"""
import sys, torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, '.')
from orientedreppoints_b200.weights import random_state_dict
from orientedreppoints_b200.detector import OrientedRepPointsDetector
from orientedreppoints_b200 import _lib
dev = torch.device('cuda'); B = int(sys.argv[1])
prec = sys.argv[2] if len(sys.argv) > 2 else 'f16x3'
depth = (sys.argv[3] if len(sys.argv) > 3 else '50')
if depth == 'swin_tiny':
    from orientedreppoints_b200.swin import random_swin_state_dict
    sd = random_swin_state_dict(0)
else:
    depth = int(depth)
    sd = random_state_dict(depth, 0, True)
det = OrientedRepPointsDetector(sd, depth, dev, prec, test_cfg=dict(score_thr=0.0))
img = torch.randint(0, 256, (B, 1024, 1024, 3), dtype=torch.uint8, device=dev)
for _ in range(3): det.forward_dense(img)

# the engine's three tensor-core entry paths, each recording (nprob, N, H, W, Cin, Cout, k, stride, algorithmic flops) of
# its call and the plan it launched
eng, launches = det.eng, []
def _conv(xs, ys, tc, cout, kh, kw, cin, stride, *a, **kw_):
    fl = sum(2.0 * y.shape[0] * y.shape[1] * y.shape[2] * cout * kh * kw * cin for y in ys)
    return (len(xs),) + tuple(xs[0].shape[:3]) + (cin, cout, kh, stride, fl)
def _splitk(x, y, tc, L, *a):
    cin = L.w_raw.shape[3]
    fl = 2.0 * y.shape[0] * y.shape[1] * y.shape[2] * L.cout * L.kh * L.kw * cin
    return (1,) + tuple(x.shape[:3]) + (cin, L.cout, L.kh, L.stride, fl)
def _stem(xs, L, n, h, w):
    return (1, n, h, w, 3, 64, 7, 2, 2.0 * n * (h // 2) * (w // 2) * 64 * 147)
def recorded(method, shape):
    fn = getattr(eng, method)
    def wrapper(*a, **kw):
        out = fn(*a, **kw)
        launches.append((shape(*a, **kw), _lib.tc_last_plan()))
        return out
    setattr(eng, method, wrapper)
for m, shape in (("_launch", _conv), ("_conv_splitk", _splitk), ("_stem_conv_s2d", _stem)):
    recorded(m, shape)

torch.cuda.synchronize(); _lib.set_timing(True); _lib.tc_timing_collect()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    det.forward_dense(img); torch.cuda.synchronize()
ms, n, fl = _lib.tc_timing_collect()
_lib.set_timing(False)
for m in ("_launch", "_conv_splitk", "_stem_conv_s2d"): delattr(eng, m)
kern = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "conv_tc_kernel" in e.name),
              key=lambda e: e.time_range.start)
assert len(kern) == len(launches) == n, (len(kern), len(launches), n)
total_us = 0.0
for i, (e, ((nprob, N, H, W, cin, cout, k, s, f), p)) in enumerate(zip(kern, launches)):
    us = e.time_range.elapsed_us()
    total_us += us
    print("tc[%3d] np=%d N=%d %4dx%-4d Cin=%4d Cout=%4d k=%d s=%d dcn=%d BN=%3d tiles=%5d grid=%3d  %8.1f us  %7.1f TFLOP/s"
          % (i, nprob, N, H, W, cin, cout, k, s, p["deform"], p["BN"], p["num_tiles"], p["grid"], us, f / (us * 1e-6) / 1e12))
print("%d conv_tc_kernel launches (torch.profiler): %.3f ms" % (len(kern), total_us * 1e-3))
print("%s %s %d tiles: %d tc launches %.3f ms, %.1f TFLOP/s algorithmic" % (prec, depth, B, n, ms, fl / ms / 1e9))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
det.capture(img.shape, img.dtype)
for _ in range(3): det.simple_test(img, return_tensors="padded")
torch.cuda.synchronize(); e0.record()
for _ in range(10): det.simple_test(img, return_tensors="padded")
e1.record(); torch.cuda.synchronize()
t = e0.elapsed_time(e1) / 10
print("%s whole step (graph + post): %.3f ms -> %.1f tiles/s" % (prec, t, B / t * 1e3))
if hasattr(det.eng, "overflow_count"): print("overflow count", det.eng.overflow_count())
