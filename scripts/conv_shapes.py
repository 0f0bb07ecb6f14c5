"""Forward and input-gradient convolution launches of the 512x512 flagship step (skip[128x5] in32 out3, skip channels 4,
bilinear, tf32).

Prints, for every tc_conv_kernel / tc_conv_patch_kernel launch of one step (plan.get_timing_records() with DIP_NO_SIDE=1,
class 0 = fprop, class 1 = dgrad), its shape, its time (CUDA events around the launch) and its rate: algorithmic
(2 * N * C * k^2 * pixels) and executed (K and N padded the way the kernel runs them: K to whole 32-channel blocks, N to
the wgmma N -- e.g. K = 160 for the 132-channel concat, N = 160 for its dgrad on the general path and 144 on the
patch path).  It also prints the bytes the launch
requests from L2 into shared memory, computed from the tile geometry of the kernel path, and that traffic's rate:
  general path (tc_conv_kernel): per tile, tap and K block one 128-pixel x 128-byte activation tile + one weight tile;
  patch path (tc_conv_patch_kernel, stride-1 3x3 on 8- or 16-wide tiles): per tile and K block one 180-pixel patch + 9
  weight tiles.
--path names the path of the libdip.so under test (the library does not report it); it defaults to patch.

usage: python scripts/conv_shapes.py [--steps N] [--path general|patch]      (DIP_LIB selects another libdip.so build)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."
H = W = 512
SCALES, CH, CS, IN_CH = 5, 128, 4, 32
NUM_SMS = 132
KB_BYTES = 128                  # one K block of one pixel: 32 fp32 channels
PATCH_BYTES = 180 * 128         # one K block of the 3x3 patch of an 8 x 16 or 16 x 8 tile


def ceil_div(a, b):
    return (a + b - 1) // b


def pick_tile(w, h):
    """tile of the general path (pick_tile in engine.cu)"""
    best = None
    for bw, bh in ((128, 1), (64, 2), (32, 4), (16, 8), (8, 16)):
        cost = ceil_div(w, bw) * bw * ceil_div(h, bh) * bh * 64 + bw + bh
        if best is None or cost < best[0]:
            best = (cost, bw, bh)
    return best[1], best[2]


def pick_nsplit(tiles, n_rows):
    sp = 1
    while sp * 2 <= 4 and tiles * sp * 2 <= NUM_SMS and n_rows % (32 * sp * 2) == 0:
        sp *= 2
    return sp


def flagship_convs():
    """(name, cls, K channels, N channels, k, out_h, out_w, kind) of every tensor-core fprop / dgrad launch.
    kind: 's1' stride-1 conv, 's2' stride-2 fprop, 'ph' 4-phase stride-2 dgrad"""
    convs = []
    for l in range(SCALES):
        Hl = H >> l
        h = Hl // 2
        cin = IN_CH if l == 0 else CH
        convs.append(("L%d down1 3x3 s2" % l, 0, cin, CH, 3, h, h, "s2"))
        if l > 0:
            convs.append(("L%d down1 dgrad (4 phases)" % l, 1, CH, cin, 3, 2 * h + 2, 2 * h + 2, "ph"))
        convs.append(("L%d down2 3x3" % l, 0, CH, CH, 3, h, h, "s1"))
        convs.append(("L%d down2 dgrad" % l, 1, CH, CH, 3, h + 2, h + 2, "s1"))
        convs.append(("L%d up 3x3" % l, 0, CH + CS, CH, 3, Hl, Hl, "s1"))
        convs.append(("L%d up dgrad" % l, 1, CH, CH + CS, 3, Hl + 2, Hl + 2, "s1"))
        convs.append(("L%d 1x1" % l, 0, CH, CH, 1, Hl, Hl, "s1"))
        convs.append(("L%d 1x1 dgrad" % l, 1, CH, CH, 1, Hl, Hl, "s1"))
    return convs


def alg_flops(cls, K, N, k, oh, ow, kind):
    """what the engine records (ConvOp::alg_flops: 2 * out pixels of the fprop * N * C * k^2, the same for its dgrad)"""
    if cls == 0:
        return 2.0 * oh * ow * N * K * k * k
    if kind == "ph":
        fo = (oh - 2) // 2
        return 2.0 * fo * fo * K * N * k * k
    fo = oh - (k - 1)
    return 2.0 * fo * fo * K * N * k * k


def executed_flops(cls, K, N, k, oh, ow, kind, path):
    kp = ceil_div(K, 32) * 32
    n_rows = ceil_div(N, 16) * 16
    nt = ceil_div(n_rows, 32) * 32
    if path == "patch" and kind == "s1" and k == 3 and pick_tile(ow, oh)[0] in (8, 16) and n_rows == 144:
        nt = 144                  # the patch path's wgmma N for the input gradient of the 132-channel concat
    if kind == "ph":
        g = oh // 2
        return 2.0 * (4 * g * g) * nt * kp * 9 / 4   # 9 taps over the 4 phases
    return 2.0 * oh * ow * nt * kp * k * k


def l2_bytes(cls, K, N, k, oh, ow, kind, path):
    kblocks = ceil_div(K, 32)
    n_rows = ceil_div(N, 16) * 16
    bw, bh = pick_tile(ow, oh)
    if path == "patch" and kind == "s1" and k == 3 and bw in (8, 16):   # the general path's tiles, one patch per K block
        tiles = ceil_div(ow, bw) * ceil_div(oh, bh)
        sp = pick_nsplit(tiles, n_rows)
        return tiles * sp * kblocks * (PATCH_BYTES + 9 * (n_rows // sp) * KB_BYTES)
    if kind == "ph":
        g = oh // 2
        bw, bh = pick_tile(g, g)
        tpp = ceil_div(g, bw) * ceil_div(g, bh)
        sp = pick_nsplit(4 * tpp, n_rows)
        return tpp * sp * 9 * kblocks * (128 * KB_BYTES + (n_rows // sp) * KB_BYTES)   # 9 taps over the 4 phases
    tiles = ceil_div(ow, bw) * ceil_div(oh, bh)
    sp = pick_nsplit(tiles, n_rows)
    return tiles * sp * k * k * kblocks * (128 * KB_BYTES + (n_rows // sp) * KB_BYTES)


def child_records(steps):
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "deep-image-prior_b200"))
    from oracle import dip_oracle as O
    import dip_engine as de
    cfg = O.SkipConfig(upsample_mode="bilinear", skip_channels=CS)
    params = [p.detach().cuda() for p in O.init_params(cfg, seed=0)]
    grads = [torch.zeros_like(p) for p in params]
    plan = de.Plan(IN_CH, 3, SCALES, CH, CS, True, H, W, precision=de.PRECISION_TF32)
    plan.bind(params, grads)
    adam = de.FusedAdam(params, lr=0.01)
    adam._bind(grads)
    z0 = torch.rand(1, IN_CH, H, W, device="cuda") * 0.1
    target = torch.rand(1, 3, H, W, device="cuda")
    out = torch.empty(1, 3, H, W, device="cuda")

    def run(n):
        de.run_iterations(plan, adam, z0, target, None, 1 / 30., 1, n, 0.01, out=out)

    run(10)
    torch.cuda.synchronize()
    plan.set_timing(True)
    run(steps)
    torch.cuda.synchronize()
    recs = plan.get_timing_records()
    plan.set_timing(False)
    print(json.dumps({"records": [list(r) for r in recs if r[0] in (0, 1)], "steps": steps}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--path", choices=("general", "patch"), default="patch")
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        child_records(args.steps)
        return
    env = dict(os.environ, DIP_NO_SIDE="1")   # kernels timed one at a time
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps)], env=env,
                         capture_output=True, text=True, check=True)
    rec = json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("{")][-1])
    per = {}
    for cls, fl, ms in rec["records"]:
        per.setdefault((cls, fl), []).append(ms)
    shapes = {}
    for c in flagship_convs():
        shapes.setdefault((c[1], alg_flops(*c[1:])), []).append(c)
    print("%-44s %8s %8s %9s %9s %8s %8s" % ("launch (%s path)" % args.path, "GFLOP", "ms", "alg TF/s", "exec TF/s", "L2 MB",
                                            "L2 GB/s"))
    tot = [0.0, 0.0, 0.0, 0.0]
    for key in sorted(per, key=lambda q: -sum(per[q])):
        cls, fl = key
        ms = sum(per[key]) / len(per[key])
        n = len(per[key]) / rec["steps"]
        cs = shapes.get(key)
        if cs is None:
            print("%-44s %8.2f %8.3f %9.1f  x%g" % ("class %d (unknown shape)" % cls, fl / 1e9, ms, fl / ms / 1e9, n))
            tot[0] += ms * n
            tot[1] += fl * n
            continue
        c = cs[0]
        exe = executed_flops(*c[1:], args.path)
        byt = l2_bytes(*c[1:], args.path)
        label = " / ".join(x[0] for x in cs)
        print("%-44s %8.2f %8.3f %9.1f %9.1f %8.1f %8.0f  x%g" % (label[:44], fl / 1e9, ms, fl / ms / 1e9, exe / ms / 1e9,
                                                                 byt / 1e6, byt / ms / 1e6, n / len(cs)))
        tot[0] += ms * n
        tot[1] += fl * n
        tot[2] += exe * n / len(cs)
        tot[3] += byt * n / len(cs)
    print("all fprop / dgrad launches: %.3f ms/step, %.1f GFLOP/step algorithmic (%.1f TFLOP/s), %.1f executed, %.0f MB L2->SM"
          % (tot[0], tot[1] / 1e9, tot[1] / tot[0] / 1e9, tot[2] / 1e9, tot[3] / 1e6))


if __name__ == "__main__":
    main()
