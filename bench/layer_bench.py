"""Per-kernel timing of the VGG-F step at the benchmark shape (B=64, 224x224): every conv layer's
fprop / dgrad / wgrad, the FC GEMMs and the memory-bound kernels, with achieved TFLOP/s or GB/s
against MEASURED_PEAKS.json, and torch (cuDNN/cuBLAS, bf16 channels_last) numbers for context.
Writes gpurun_out/layer_bench.json and prints a table."""
# Without MEASURED_PEAKS.json the peaks are the H100 SXM data sheet's: 989 dense bf16 TFLOP/s and
# 3,350 GB/s.  Every native conv call uses the training step's kernel choice (bn = 0, ksplit = 0);
# where the output side of a conv has >= 256 channels (the only place the width rule can pick a
# 256-wide tile) the same call is also timed at bn = 128 and bn = 256, rows tagged "[bn=...]".
# The table is headed by the card's name, power limit and maximum SM clock.
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.models.vggf import vggf_spec

dev = "cuda"
B = int(os.environ.get("LB_BATCH", "64"))
HW = 224
PEAK = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) \
    if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"bf16_tflops": 989.0, "hbm_gbs": 3350.0}
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def card_info():
    info = {"name": torch.cuda.get_device_name(), "power_limit": None, "sm_max_clock": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit"], info["sm_max_clock"] = q[0].strip(), q[1].strip()
    except (OSError, IndexError, subprocess.SubprocessError):
        pass
    return info


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()                      # evict L2 between timed launches
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


rows = []
spec = vggf_spec(3)
h = HW
with_torch = os.environ.get("LB_TORCH", "1") == "1"
for i, c in enumerate(spec.convs):
    if i == 0:
        M = B * h * h
        col = torch.randn(M, 64, device=dev).bfloat16()
        w0 = torch.randn(64, 64, device=dev).bfloat16()
        b0 = torch.randn(64, device=dev)
        y0 = torch.empty(M, 64, dtype=torch.bfloat16, device=dev)
        dz0 = torch.randn(M, 64, device=dev).bfloat16()
        dw0 = torch.zeros(64, 64, device=dev)
        t = timeit(lambda: ops.gemm(col, w0, y0, M=M, N=64, K=64, epi="bf16_bias_relu", bias=b0, bn=64))
        rows.append(("conv0 fprop(im2col gemm)", t, 2.0 * M * 64 * 27 / 1e12, (M * 64 * 2 * 2) / 1e9))
        t = timeit(lambda: ops.gemm(dz0, col, dw0, M=64, N=64, K=M, a_mn=True, b_mn=True, epi="f32_atomic", ksplit=296, ldo=64))
        rows.append(("conv0 wgrad(gemm)", t, 2.0 * M * 64 * 27 / 1e12, (M * 64 * 2 * 2) / 1e9))
        x4 = torch.randn(B, h, h, 4, device=dev).bfloat16()
        yy = torch.empty(B, h, h, 64, dtype=torch.bfloat16, device=dev)
        Cx = ops.require()
        t = timeit(lambda: Cx.conv0_fprop(x4, w0, b0, yy))
        rows.append(("conv0 fprop fused (no im2col)", t, 2.0 * M * 64 * 27 / 1e12, (M * 64 * 2) / 1e9))
        t = timeit(lambda: Cx.conv0_wgrad(dz0.view(B, h, h, 64), x4, dw0))
        rows.append(("conv0 wgrad fused (no im2col)", t, 2.0 * M * 64 * 27 / 1e12, (M * 64 * 2) / 1e9))
        del col, y0, dz0, x4, yy
    else:
        x = torch.randn(B, h, h, c.cin, device=dev).bfloat16()
        w = (torch.randn(c.cout, 3, 3, c.cin, device=dev) * 0.05).bfloat16()
        bias = torch.randn(c.cout, device=dev)
        y = torch.empty(B, h, h, c.cout, dtype=torch.bfloat16, device=dev)
        dz = torch.randn(B, h, h, c.cout, device=dev).bfloat16()
        dx = torch.empty_like(x)
        dw = torch.zeros(c.cout, 3, 3, c.cin, device=dev)
        fl = 2.0 * B * h * h * c.cout * 9 * c.cin / 1e12
        C = ops.require()

        def timed(name, wide, fn):               # fn(bn)
            rows.append((name, timeit(lambda: fn(0)), fl, 0))
            if wide:
                for bn in (128, 256):
                    rows.append(("%s [bn=%d]" % (name, bn), timeit(lambda: fn(bn)), fl, 0))

        timed("%s fprop %dx%d %d->%d" % (c.name, h, h, c.cin, c.cout), c.cout >= 256,
              lambda bn: C.conv_fprop(x, w, bias, y, True, bn))
        if c.pool_after:                         # what the step runs for a pooled layer
            pooled = torch.empty(B, h // 2, h // 2, c.cout, dtype=torch.bfloat16, device=dev)
            pmask = ops.pool_mask_like(B, h, h, c.cout, dev)
            timed("%s fprop+pool" % c.name, c.cout >= 256, lambda bn: C.conv_fprop_pool(x, w, bias, pooled, pmask, bn))
        timed("%s dgrad" % c.name, c.cin >= 256, lambda bn: C.conv_dgrad(dz, w, x, dx, None, bn))
        cs = torch.zeros(c.cin, device=dev)
        timed("%s dgrad+colsum" % c.name, c.cin >= 256, lambda bn: C.conv_dgrad(dz, w, x, dx, cs, bn))
        # Cin = 64 on 8-divisible maps: the halo kernel
        timed("%s wgrad" % c.name, c.cin >= 256, lambda bn: C.conv_wgrad(dz, x, dw, 1.0, 0, bn))
        if with_torch:
            xt = x.permute(0, 3, 1, 2)            # NCHW view, channels_last memory
            wt = w.permute(0, 3, 1, 2)
            t = timeit(lambda: F.conv2d(xt, wt, None, padding=1))
            rows.append(("%s fprop cuDNN bf16" % c.name, t, fl, 0))
            dzt = dz.permute(0, 3, 1, 2)
            t = timeit(lambda: torch.ops.aten.convolution_backward(dzt, xt, wt, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False]))
            rows.append(("%s dgrad cuDNN bf16" % c.name, t, fl, 0))
            t = timeit(lambda: torch.ops.aten.convolution_backward(dzt, xt, wt, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False]))
            rows.append(("%s wgrad cuDNN bf16" % c.name, t, fl, 0))
        if c.pool_after:
            p = torch.empty(B, h // 2, h // 2, c.cout, dtype=torch.bfloat16, device=dev)
            t = timeit(lambda: ops.maxpool2x2(y, out=p))
            rows.append(("%s maxpool fwd" % c.name, t, 0, y.numel() * 2 * 1.25 / 1e9))
            t = timeit(lambda: ops.maxpool2x2_relu_bwd(y, p, out=dz))
            rows.append(("%s pool+relu bwd" % c.name, t, 0, y.numel() * 2 * 2.25 / 1e9))
            cs2 = torch.zeros(c.cout, device=dev)
            t = timeit(lambda: ops.maxpool2x2_relu_bwd(y, p, out=dz, colsum=cs2))
            rows.append(("%s pool+relu bwd+colsum" % c.name, t, 0, y.numel() * 2 * 2.25 / 1e9))
        t = timeit(lambda: ops.bias_grad(dz.view(-1, c.cout), torch.zeros(c.cout, device=dev), B * h * h, c.cout))
        rows.append(("%s bias_grad" % c.name, t, 0, dz.numel() * 2 / 1e9))
        del x, y, dz, dx
    if c.pool_after:
        h //= 2

# FC stack
for f in spec.fcs:
    W = (torch.randn(f.fout, f.fin, device=dev) * 0.01).bfloat16()
    X = torch.randn(B, f.fin, device=dev).bfloat16()
    ld = (f.fout + 7) // 8 * 8
    dY = torch.randn(B, ld, device=dev).bfloat16()
    acc = torch.zeros(B, f.fout, device=dev)
    dacc = torch.zeros(B, f.fin, device=dev)
    dW = torch.zeros(f.fout, f.fin, device=dev)
    mt = (f.fout + 127) // 128
    ks = max(1, min((f.fin + 63) // 64, 256 // mt))
    t = timeit(lambda: ops.gemm(W, X, acc, M=f.fout, N=B, K=f.fin, epi="f32_atomic_t", ksplit=ks, ldo=f.fout))
    rows.append(("%s fwd gemm ks%d" % (f.name, ks), t, 2.0 * B * f.fin * f.fout / 1e12, W.numel() * 2 / 1e9))
    t = timeit(lambda: ops.gemm(dY, X, dW, M=f.fout, N=f.fin, K=B, a_mn=True, b_mn=True, epi="f32_store", ldo=f.fin))
    rows.append(("%s wgrad gemm" % f.name, t, 2.0 * B * f.fin * f.fout / 1e12, W.numel() * 4 / 1e9))
    mt = (f.fin + 127) // 128
    ks = max(1, min((f.fout + 63) // 64, 256 // mt))
    t = timeit(lambda: ops.gemm(W, dY, dacc, M=f.fin, N=B, K=f.fout, a_mn=True, epi="f32_atomic_t" if ks > 1 else "f32_store_t", ksplit=ks, ldo=f.fin))
    rows.append(("%s dgrad gemm ks%d" % (f.name, ks), t, 2.0 * B * f.fin * f.fout / 1e12, W.numel() * 2 / 1e9))

# optimizer + augment
n = 136_400_000 // 4 * 4
p, m, v, g = (torch.zeros(n, device=dev) for _ in range(4))
sh = torch.zeros(n, dtype=torch.bfloat16, device=dev)
t = timeit(lambda: ops.adam_step(p, m, v, g32=g, shadow=sh, lr=1e-3, step=1, zero=g))
rows.append(("adam fused (136M, fp32 grad)", t, 0, n * (4 * 4 + 3 * 4 + 2 + 4) / 1e9))
src = torch.randint(0, 255, (B, 128, 128, 3), dtype=torch.uint8, device=dev)
from distributed_vgg_f_b200.data import transforms as T
prm = T.sample_train_params(B, 128, 128).to(dev)
col = torch.empty(B * HW * HW, 64, dtype=torch.bfloat16, device=dev)
t = timeit(lambda: ops.augment(src, prm, col, (256, 256), mode="im2col", pad=64))
rows.append(("augment -> im2col (one pass)", t, 0, col.numel() * 2 / 1e9))
x4 = torch.empty(B, HW, HW, 4, dtype=torch.bfloat16, device=dev)
t = timeit(lambda: ops.augment(src, prm, x4, (256, 256), mode="nhwc", pad=4))
rows.append(("augment -> NHWC4", t, 0, x4.numel() * 2 / 1e9))
t = timeit(lambda: ops.require().im2col_c3(x4, col, 64))
rows.append(("NHWC4 -> im2col", t, 0, col.numel() * 2 / 1e9))

out = []
card = card_info()
print("card: %s, power limit %s, max SM clock %s; peaks %.0f TFLOP/s, %.0f GB/s"
      % (card["name"], card["power_limit"], card["sm_max_clock"], PEAK["bf16_tflops"], PEAK["hbm_gbs"]))
print("%-46s %9s %9s %9s %7s" % ("kernel", "ms", "TFLOP/s", "GB/s", "%peak"))
for name, ms, tf, gb in rows:
    tfs = tf / (ms / 1e3) if tf else 0.0
    gbs = gb / (ms / 1e3) if gb else 0.0
    frac = tfs / PEAK["bf16_tflops"] if tf else (gbs / PEAK["hbm_gbs"] if gb else 0)
    print("%-46s %9.3f %9.1f %9.1f %6.1f%%" % (name, ms, tfs, gbs, 100 * frac))
    out.append({"kernel": name, "ms": ms, "tflops": tfs, "gbs": gbs, "frac_of_measured_peak": frac})
os.makedirs("gpurun_out", exist_ok=True)
json.dump({"batch": B, "peaks": PEAK, "rows": out}, open("gpurun_out/layer_bench.json", "w"), indent=1)
