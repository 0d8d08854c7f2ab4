"""Golden vectors for convex_giou (tests/golden/convex_giou_ref.npz) from the reference's OWN device code:
mmdet/ops/iou/src/convex_giou_kernel.cu up to `__global__ void convex_giou_kernel` (devrIoU :730-804 and everything it
calls) is compiled as host C++ the way oracle/build_ref.py compiles the other CUDA-only ops (read where it lies, never
written to disk, separately rounded arithmetic), behind the C-ABI loop HARNESS below, into a temporary directory.

The reference reads an uninitialised point where one clip endpoint lies within 1e-8 of the cut line and the other within
1e-8 of the first (polygon_cut / lineCross :176-211), so its result is undefined there.  To keep such pairs out of the
golden, the reference is also built at -O0 twice, with every uninitialised automatic variable set to zero and to a
pattern (-ftrivial-auto-var-init); a pair is kept only if both builds and the -O2 build agree bit for bit.  The script
prints how many pairs that drops.

    python tests/golden/gen_golden_convex_giou.py      # needs the reference tree ($ORP_REFERENCE_ROOT)
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import REF, _DEVICE_PREFIX                                     # noqa: E402
from orientedreppoints_b200.synth import gen_rotated_boxes                            # noqa: E402

SRC = os.path.join(REF, "mmdet/ops/iou/src/convex_giou_kernel.cu")
CUT = "__global__ void convex_giou_kernel"
HARNESS = r'''
extern "C" void ref_convex_giou(const float *p, const float *q, int n, float *out)
{
    for (int i = 0; i < n; ++i) out[19 * i + 18] = devrIoU(p + 18 * i, q + 8 * i, out + 19 * i, i);
}
'''
BUILDS = {"o2": ["-O2"], "zero": ["-O0", "-ftrivial-auto-var-init=zero"], "pattern": ["-O0", "-ftrivial-auto-var-init=pattern"]}


def build(tmp):
    text = open(SRC).read()
    body = "\n".join(l for l in text[:text.index(CUT)].splitlines() if not l.lstrip().startswith("#include"))
    libs = {}
    for name, flags in BUILDS.items():
        so = os.path.join(tmp, "ref_convex_giou_%s.so" % name)
        cmd = ["g++", "-x", "c++", "-", "-shared", "-fPIC", "-w", "-ffp-contract=off", "-o", so] + flags
        subprocess.run(cmd, input=(_DEVICE_PREFIX + body + "\n" + HARNESS).encode(), check=True)
        libs[name] = ctypes.CDLL(so)
    return libs


def run(lib, p, q):
    p = np.ascontiguousarray(p, np.float32)
    q = np.ascontiguousarray(q, np.float32)
    out = np.zeros((len(p), 19), np.float32)
    vp = ctypes.c_void_p
    lib.ref_convex_giou(vp(p.ctypes.data), vp(q.ctypes.data), len(p), vp(out.ctypes.data))
    return out


def _rot(th):
    c, s = np.cos(th), np.sin(th)
    return np.stack([np.stack([c, -s], -1), np.stack([s, c], -1)], -2)               # [..., 2, 2]


def cases():
    """(kind, pts [n,18] float32, quads [n,8] float32)"""
    rng = np.random.RandomState(0)
    out = []

    def quads_of(n, seed, extent):
        return gen_rotated_boxes(n, seed=seed, extent=extent)[:, :8].astype(np.float64)

    def scatter(q, spread, shift, rng):
        """9 points in a box of the quad's size times `spread`, rotated, shifted by `shift` quad sizes"""
        n = len(q)
        c = q.reshape(n, 4, 2).mean(1)
        u, v = q[:, 2:4] - q[:, 0:2], q[:, 6:8] - q[:, 0:2]
        size = np.sqrt(np.abs(u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]))[:, None]
        local = (rng.rand(n, 9, 2) - 0.5) * size[:, None, :] * spread[:, None, :]
        local = np.einsum("nij,nkj->nki", _rot(rng.uniform(-np.pi, np.pi, n)), local)
        d = rng.normal(0, 1, (n, 2))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        return (c[:, None, :] + local + (d * shift[:, None] * size)[:, None, :]).reshape(n, 18)

    # realistic: SURVEY 8(d) quads up to 4000 px, point sets of random spread and offset -> IoU over 0..1
    n = 1600
    q = quads_of(n, 11, 4000.0)
    p = scatter(q, rng.uniform(0.3, 1.8, (n, 2)), rng.uniform(0.0, 0.8, n), rng)
    out.append(("realistic", p, q))
    # disjoint: GIoU < 0
    n = 300
    q = quads_of(n, 12, 4000.0)
    out.append(("disjoint", scatter(q, rng.uniform(0.3, 1.0, (n, 2)), rng.uniform(2.0, 6.0, n), rng), q))
    # the point set contains the quad / lies inside it
    n = 200
    q = quads_of(n, 13, 1024.0)
    out.append(("contains", scatter(q, np.full((n, 2), 4.0), np.zeros(n), rng), q))
    c = q.reshape(n, 4, 2).mean(1)
    w = rng.uniform(0.05, 0.9, (n, 9, 1))
    inside = c[:, None, :] + (q.reshape(n, 4, 2)[:, rng.randint(0, 4, 9), :] - c[:, None, :]) * w
    out.append(("inside", inside.reshape(n, 18), q))
    # both quad orientations
    n = 300
    q = quads_of(n, 14, 1024.0)
    p = scatter(q, rng.uniform(0.5, 1.5, (n, 2)), rng.uniform(0.0, 0.5, n), rng)
    out.append(("quad_ccw", p, q))
    out.append(("quad_cw", p, q.reshape(n, 4, 2)[:, ::-1, :].reshape(n, 8)))
    # quad corners equal to points of the set (the de-duplication before the union hull)
    n = 300
    q = np.round(quads_of(n, 15, 1024.0))
    p = scatter(q, rng.uniform(0.3, 1.2, (n, 2)), rng.uniform(0.0, 0.3, n), rng)
    k = rng.randint(1, 5, n)
    for i in range(n):
        slots = rng.permutation(9)[:k[i]]
        corners = rng.permutation(4)[:k[i]]
        for s, cc in zip(slots, corners):
            p[i, 2 * s:2 * s + 2] = q[i, 2 * cc:2 * cc + 2]
    out.append(("shared_corners", p, q))
    # duplicated input points
    n = 200
    q = quads_of(n, 16, 1024.0)
    p = scatter(q, rng.uniform(0.5, 1.5, (n, 2)), rng.uniform(0.0, 0.5, n), rng)
    for i in range(n):
        src, dst = rng.randint(0, 9, 3), rng.randint(0, 9, 3)
        for s, d in zip(src, dst):
            p[i, 2 * d:2 * d + 2] = p[i, 2 * s:2 * s + 2]
    out.append(("duplicated", p, q))
    # collinear and all-equal sets (hull of fewer than three vertices)
    n = 100
    q = quads_of(n, 17, 256.0)
    c = q.reshape(n, 4, 2).mean(1)
    t = rng.uniform(-30, 30, (n, 9, 1))
    d = _rot(rng.uniform(-np.pi, np.pi, n))[:, :, 0]
    out.append(("collinear", (c[:, None, :] + t * d[:, None, :]).reshape(n, 18), q))
    ti = np.round(t)
    out.append(("collinear_int", (np.round(c)[:, None, :] + ti * np.array([1.0, 2.0])).reshape(n, 18), q))
    out.append(("all_equal", np.tile(c + rng.normal(0, 5, (n, 2)), (1, 9)), q))
    # the degenerate point sets and quads of geometry_edges.npz, every combination
    e = np.load(os.path.join(HERE, "geometry_edges.npz"))
    mp, cq = e["mar_pts"].astype(np.float64), e["cx_quads"].astype(np.float64)
    out.append(("edges", np.repeat(mp, len(cq), 0), np.tile(cq, (len(mp), 1))))
    return [(k, p.astype(np.float32), q.astype(np.float32)) for k, p, q in out]


def main():
    with tempfile.TemporaryDirectory() as tmp:
        libs = build(tmp)
        kinds, P, Q, O = [], [], [], []
        for kind, p, q in cases():
            res = {name: run(lib, p, q) for name, lib in libs.items()}
            bits = [r.view(np.int32) for r in res.values()]
            keep = np.ones(len(p), bool)
            for b in bits[1:]:
                keep &= (b == bits[0]).all(1)
            print("%-16s %5d pairs, %d dropped (result depends on uninitialised memory)" % (kind, len(p), (~keep).sum()))
            kinds += [kind] * int(keep.sum())
            P.append(p[keep]); Q.append(q[keep]); O.append(res["o2"][keep])
    P, Q, O = np.concatenate(P), np.concatenate(Q), np.concatenate(O)
    g = O[:, 18]
    print("%d pairs, giou in [%.3f, %.3f], %d < 0, %d rows with NaN" % (len(P), np.nanmin(g), np.nanmax(g), (g < 0).sum(),
                                                                       np.isnan(O).any(1).sum()))
    np.savez_compressed(os.path.join(HERE, "convex_giou_ref.npz"), pts=P, quads=Q, out=O, kind=np.array(kinds))


if __name__ == "__main__":
    main()
