"""Writes docs/KERNELS.md: every __global__ kernel of the native library with what it replaces in the reference,
its footprint (registers / static shared memory from cuobjdump --dump-resource-usage, threads from the launch
code) and the Hopper-specific instructions in its SASS (sass_out/INDEX.md).  CPU box:
    python build_native.py && bash bench/dump_sass.sh && python bench/kernel_catalog.py"""
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROLE = [   # (regex on the demangled name, role, what it replaces in the reference)
    (r"conv_halo_kernel<\d+, false", "conv fprop, 224² / 112² layers: halo tile once per channel chunk, nine taps = nine descriptor views; bias + ReLU (+ fused 2×2 max-pool) epilogue", "cuDNN conv fwd + ATen relu (+ max_pool2d) — `distributedVggf.py:162`"),
    (r"conv_halo_kernel<\d+, true", "conv dgrad, 224² / 112² layers; previous layer's ReLU mask + bias gradient in the epilogue", "cuDNN dgrad + threshold_backward — `:171`"),
    (r"umma_kernel<b200::ConvPolicy<\d+, \d+, false", "conv fprop, 56² … 14² layers: implicit GEMM, 4-D TMA boxes per tap, register accumulators in two consumer warpgroups; bias + ReLU (+ pool) epilogue", "cuDNN conv fwd — `:162`"),
    (r"umma_kernel<b200::ConvPolicy<\d+, \d+, true", "conv dgrad, 56² … 14² layers (weights read MN-major, mirrored taps)", "cuDNN dgrad — `:171`"),
    (r"umma_kernel<b200::WgradPolicy", "conv wgrad: both operands MN-major 4-D TMA boxes, split-K over pixel tiles, `red.global.add` straight into the gradient arena", "cuDNN wgrad — `:171`"),
    (r"wgrad_halo64_kernel", "conv wgrad for Cin = 64 (one X halo serves all nine taps, two taps stacked along M)", "cuDNN wgrad — `:171`"),
    (r"conv0_kernel<false>|conv0_kernel<0>", "first conv (K = 27) fprop: im2col operand built in shared memory from NHWC4 pixels, wgmma", "cuDNN conv fwd — `:162`"),
    (r"conv0_kernel<true>|conv0_kernel<1>", "first conv wgrad (same shared-memory operand, MN-major)", "cuDNN wgrad — `:171`"),
    (r"umma_kernel<b200::GemmPolicy", "FC GEMMs: swap-AB split-K forward / dgrad, wgrad with epilogue → fp32 arena or `bf16(dW/ws)` straight into the symmetric wire", "cuBLAS SGEMM under `nn.Linear` — `:162`, `:171`"),
    (r"head_ce_kernel", "K-FUN2+CE: last Linear + log-softmax / NLL + metrics + dlogits + the layer's dW, db, dX in one launch", "cuBLAS + ATen log_softmax / nll_loss + `Accuracy2` / `Average` — `:56`, `:168`, `distributedUtil.py:95-96`"),
    (r"head_ce_kd_kernel", "K-FUN2+CE with knowledge distillation: head_ce_kernel's launch, the teacher's logits read too; loss (1 − α) CE + α T² KL and its dlogits", "`F.cross_entropy` + `F.kl_div` of a distillation script — not in the reference"),
    (r"tta_accumulate_kernel", "--val-tta view-mean reduction: each view's softmax added into an fp32 [B][C] accumulator in view order; at the last view -log of the label's mean probability and its argmax into the meter", "the mean softmax of torchvision's `ten_crop` / `five_crop` views — not in the reference"),
    (r"class_metrics_kernel", "--val-metrics: per evaluation batch, int64 confusion-matrix counts of (label, first maximum of the logits or of the --val-tta view mean) and the count of labels ranked in the top 5; integer atomics", "scikit-learn `confusion_matrix` / torchvision's Acc@5 — not in the reference"),
    (r"cross_entropy_kd_kernel", "cross-entropy with knowledge distillation for heads that do not fuse (C > 8, B > 256, VGG-16)", "`F.cross_entropy` + `F.kl_div` of a distillation script — not in the reference"),
    (r"cross_entropy_kernel", "cross-entropy fwd + bwd + metrics for wide heads (VGG-16/1000)", "`F.cross_entropy` — `:168`"),
    (r"fc_bias_act_kernel", "FC epilogue: bias + ReLU + Philox dropout → bf16 (mask never stored)", "ATen bias/relu/dropout — `:52-57`"),
    (r"fc_grad_act_kernel", "FC backward epilogue: ReLU / dropout mask regenerated from the activation", "ATen threshold_backward / dropout backward"),
    (r"bias_grad", "bias gradients that no GEMM / pool epilogue already produced", "autograd sum"),
    (r"maxpool2x2_fwd_kernel|maxpool2x2_relu_bwd_kernel|maxpool2x2_relu_bwd_odd_kernel", "un-fused max-pool fwd / ReLU + pool bwd (tile shapes the epilogue cannot pool, odd maps in floor mode, `B200_FUSE_POOL=0`)", "cuDNN / ATen max_pool2d"),
    (r"unpool2x2_kernel", "backward of the epilogue-fused pool: pooled gradient + argmax bit masks → full-resolution dz, bias gradient fused", "max_pool2d_backward + threshold_backward"),
    (r"adaptive_avgpool", "AdaptiveAvgPool2d(7,7) fwd / bwd (elided when the map is already 7×7)", "ATen adaptive_avg_pool2d — torchvision VGG"),
    (r"augment_view_nhwc_kernel", "--val-tta: one view (five-crop corner, centre, or mirror) of the fused transform: uint8 HWC → normalised bf16 NHWC4", "torchvision `FiveCrop` / `TenCrop` after `Resize` — not in the reference"),
    (r"augment_ragged_views_h_kernel", "--val-tta, images of any size: Pillow's horizontal pass once over the union of the rows and columns every view reads", "PIL `Resize` before `TenCrop` — not in the reference"),
    (r"augment_ragged_view_v_kernel", "--val-tta, images of any size: Pillow's vertical pass and the view's crop, per view", "PIL `Resize` + `TenCrop` — not in the reference"),
    (r"jpeg_idct_kernel", "--pipeline stream: dequantise + JDCT_ISLOW IDCT of every 8×8 coefficient block of the batch into uint8 sample planes, libjpeg's range-limit table", "PIL `Image.open` (libjpeg-turbo IDCT) — `:88-95`, `:103-108`"),
    (r"jpeg_color_kernel", "--pipeline stream: libjpeg's fancy chroma upsampling and fixed-point YCbCr → RGB, each image at its geometry offset; raw members copied", "PIL `convert(\"RGB\")` (libjpeg-turbo upsampling and colour conversion)"),
    (r"augment_nhwc_kernel|augment_im2col_kernel", "the six PIL transforms as one coordinate chain per output pixel: uint8 HWC → normalised bf16 NHWC4", "PIL / torchvision transforms — `:88-95`, `:103-108`"),
    (r"im2col3x3_c3_kernel|nchw_f32_to_nhwc_bf16_kernel", "input layout conversion for float inputs (tests, `forward_logits`)", "—"),
    (r"adam_kernel", "fused Adam over a bucket: grad (fp32 arena or bf16 wire) → fp32 master, moments, bf16 shadow, gradient range re-zeroed; evict-first streams", "`torch.optim.Adam` foreach kernels + `zero_grad` — `:230`, `:170-172`"),
    (r"sgd_kernel", "fused SGD + momentum (the reference's vestigial constants)", "—"),
    (r"layerwise_norms_kernel", "LAMB / LARS phase 1 over a bucket: LAMB's moments, and per-CTA partial sums of ‖p‖² and ‖u‖² (LAMB) or ‖g‖² (LARS) at host-assigned slots, one tensor per CTA", "timm `Lamb` / `Lars`: per-tensor `norm` — not in the reference"),
    (r"layerwise_update_kernel", "LAMB / LARS phase 2 over the tensors a bucket completes: trust ratio from the slots in a fixed order, the update, bf16 shadow, EMA, (LARS) gradient re-zeroed", "timm `Lamb` / `Lars` `step` — not in the reference"),
    (r"allreduce_kernel<0", "K-AR one-shot: every rank sums all peers' chunk over peer memory (no-multicast fallback)", "c10d Reducer + gloo all-reduce — `:225`, `:171`"),
    (r"allreduce_kernel<1", "K-AR two-shot: reduce-scatter + all-gather by peer loads / stores in one pass", "same"),
    (r"allreduce_kernel<2", "K-AR NVLS: pack fp32→bf16·1/ws, handshake, `multimem.ld_reduce` (switch adds, fp32 accumulate) + `multimem.st`, handshake", "same"),
    (r"zero1_kernel", "fused ZeRO-1 step: reduce-scatter → Adam on owned cells → all-gather of the new bf16 weights, one launch per FC bucket", "Reducer + all-reduce + `Adam.step` — `:171-172`"),
    (r"broadcast_kernel", "K-BCAST: rank 0's parameters pulled over NVLink through the wire buffer", "DDP constructor `_sync_module_states` — `:225`"),
    (r"barrier_kernel", "device-side barrier (tests)", "—"),
    (r"cast_", "fp32 ↔ bf16 casts (start-up: master → shadow)", "—"),
    (r"psgd_project_kernel", "PowerSGD: M = g/k′ + e over the error arena and P = M·Q, one row per CTA", "`powerSGD_hook`: error add + `torch.bmm`"),
    (r"psgd_backproject_kernel", "PowerSGD: Q = Mᵀ·P per row split (added in order by splitk_reduce)", "`powerSGD_hook`: `torch.bmm`"),
    (r"psgd_orthogonalize_kernel", "PowerSGD: modified Gram–Schmidt of P or Q, one CTA per matrix", "`powerSGD_hook`: `_orthogonalize`"),
    (r"psgd_decompress_kernel", "PowerSGD: G = P·Qᵀ/W over the gradient, e = M − G", "`powerSGD_hook`: `torch.bmm` + error store"),
]


def main():
    res = {}
    for o in sorted(glob.glob(os.path.join(ROOT, "build", "obj", "*.cu.o"))):
        out = subprocess.run(["cuobjdump", "--dump-resource-usage", o], capture_output=True, text=True).stdout
        fn = None
        for line in out.splitlines():
            m = re.match(r"\s*Function (\S+):", line)
            if m:
                fn = m.group(1)
                continue
            m = re.search(r"REG:(\d+).*?SHARED:(\d+)", line)
            if m and fn:
                name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()
                name = re.sub(r"\((?:[^()]|\([^()]*\))*\)$", "", name).replace("CUtensorMap_st", "TMap")
                res[name] = (os.path.basename(o)[:-5], int(m.group(1)), int(m.group(2)))
                fn = None
    index = {}
    p = os.path.join(ROOT, "sass_out", "INDEX.md")
    if os.path.exists(p):
        for line in open(p):
            m = re.match(r"\| (\S+) \| `(.+?)` \| (\d+) \| (.*) \|", line)
            if m:
                index[m.group(2)] = (int(m.group(3)), m.group(4))
    rows = []
    for name, (tu, regs, smem) in sorted(res.items(), key=lambda kv: (kv[1][0], kv[0])):
        role, repl = next(((r, rp) for pat, r, rp in ROLE if re.search(pat, name)), ("(unclassified)", "—"))
        key = next((k for k in index if k.rstrip() == name[:110].rstrip()), None)
        n_sass, mn = index.get(key, (0, ""))
        rows.append((tu, name, regs, smem, n_sass, mn, role, repl))
    with open(os.path.join(ROOT, "docs", "KERNELS.md"), "w") as f:
        f.write("# Kernel catalogue (generated by bench/kernel_catalog.py from the sm_90a objects)\n\n"
                "Every `__global__` function of `distributed_vgg_f_b200/_C*.so`: what it does, which library call of the reference it "
                "stands in for (lines of `distributedVggf.py` / `distributedUtil.py`), registers per thread and static shared memory "
                "(`cuobjdump --dump-resource-usage`; the wgmma kernels add up to 227 KB of dynamic shared memory at launch), SASS size "
                "and its Hopper-specific mnemonics (`sass_out/INDEX.md`).  Template instantiations are listed individually.\n\n"
                "| TU | kernel | regs | static smem | SASS instr. | native mnemonics | role | replaces |\n|---|---|---|---|---|---|---|---|\n")
        for tu, name, regs, smem, n_sass, mn, role, repl in rows:
            f.write("| %s | `%s` | %d | %d | %d | %s | %s | %s |\n" % (tu, name[:100], regs, smem, n_sass, mn, role, repl))
    print("kernels:", len(rows), "unclassified:", sum(1 for r in rows if r[6] == "(unclassified)"))


if __name__ == "__main__":
    main()
