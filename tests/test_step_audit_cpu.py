"""The bookkeeping of the step audit (step_audit.py) on CPU tensors, without the extension.

``_MiniEngine`` replays the launch sequence of ``NativeEngine`` (fused pool, fused head, Adam, one
optimizer bucket per parameter) for a four-conv network on CPU tensors, through ``step_audit._Proxy``
and a scripted fake extension that only writes recognisable bytes into what each kernel writes.
A clean sequence (two training steps, an evaluation step, a group of two micro-batches) must pass;
each planted defect must fail with a message naming it.
"""
import types

import pytest
import torch

import launch_replay as LR
import step_audit as SA
from distributed_vgg_f_b200.models.vggf import ConvSpec, FCSpec, VGGSpec

B, HW = 2, 4
SPEC = VGGSpec(convs=(ConvSpec("features.0", 3, 64, False), ConvSpec("features.2", 64, 64, True),
                      ConvSpec("features.5", 64, 64, False), ConvSpec("features.7", 64, 64, True)),
               fcs=(FCSpec("classifier.0", 64, 16, True, 0.5), FCSpec("classifier.3", 16, 3, False, 0.0)),
               num_classes=3, pooled_hw=1)


class _FakeC:
    """Each kernel writes a new value into every argument it stores, adds 1 to what it accumulates,
    and clears (or, optimizer state, increments) what it updates."""
    EPI_F32_STORE, EPI_F32_ATOMIC, EPI_F32_ATOMIC_T, EPI_BF16_BIAS_RELU, EPI_F32_STORE_T, EPI_BF16_STORE = range(6)

    def __init__(self):
        self.n = 0
        self._roles = types.SimpleNamespace(C=self)

    def __getattr__(self, name):
        if name not in LR.RECORDED:
            raise AttributeError(name)

        def kernel(*args):
            tensors, sc = LR.split_args(name, args)
            if name in ("adam", "sgd"):
                sc["_zero_is_g32"] = tensors["zero"] is tensors["g32"]
            for key, t in tensors.items():
                if t is None:
                    continue
                role = SA.Auditor._role(self._roles, name, key, sc)
                self.n += 1
                if role == LR.STORE:
                    t.fill_(self.n % 97 + 1)
                elif role == LR.ACCUM:
                    t.add_(1)
                elif role == LR.UPDATE:
                    t.zero_() if key in ("acc", "zero", "g32") else t.add_(1)
        return kernel


class _MiniEngine:
    def __init__(self, defect=None):
        self.defect = defect
        sizes = {}
        for c in SPEC.convs:
            sizes[c.name + ".weight"] = c.cout * 9 * c.cin if c.cin != 3 else 64 * 64
            sizes[c.name + ".bias"] = c.cout
        for f in SPEC.fcs:
            sizes[f.name + ".weight"], sizes[f.name + ".bias"] = f.fout * f.fin, f.fout
        self.off, n = {}, 0
        for name in SPEC.param_names:
            self.off[name] = (n, n + sizes[name])
            n += sizes[name]
        self.p32, self.g32, self.m32, self.v32 = (torch.zeros(n) for _ in range(4))
        self.p32.normal_()
        self.w16 = self.p32.to(torch.bfloat16)
        bf = torch.bfloat16
        self.src = [torch.zeros(B, 8, 8, 3, dtype=torch.uint8) for _ in range(2)]
        self.prm = [torch.zeros(B, 8) for _ in range(2)]
        self.lab = [torch.zeros(B, dtype=torch.int64) for _ in range(2)]
        self.slot = 0
        self.x = torch.zeros(B, HW, HW, 4, dtype=bf)
        self.acts, self.pools, self.masks, h = [], [], [], HW
        for c in SPEC.convs:
            self.acts.append(torch.empty(B, h, h, c.cout, dtype=bf))
            if c.pool_after:
                h //= 2
            self.pools.append(torch.empty(B, h, h, c.cout, dtype=bf) if c.pool_after else None)
            self.masks.append(torch.zeros(B, h, h, c.cout // 32, 4, dtype=torch.int32) if c.pool_after else None)
        self.fc_acc, self.fc_y = torch.zeros(B, 16), torch.empty(B, 16, dtype=bf)
        self.fc_dacc, self.dfeat = torch.zeros(B, 64), torch.empty(B, 1, 1, 64, dtype=bf)
        self.fc_dz = [torch.zeros(B, 16, dtype=bf), torch.zeros(B, 8, dtype=bf)]
        self.logits, self.meter, self.loss = torch.zeros(B, 3), torch.zeros(4), torch.zeros(1)
        self.dbuf = [torch.empty(B * HW * HW * 64, dtype=bf) for _ in range(2)]
        params = {n: (self.v(self.w16 if n.endswith(".weight") else self.p32, n), self.v(self.g32, n))
                  for n in SPEC.param_names}
        initial = [(self.p32, "parameters"), (self.w16, "weight shadow"), (self.m32, "zeros"), (self.v32, "zeros"),
                   (self.g32, "zeros"), (self.fc_acc, "zeros"), (self.fc_dacc, "zeros"), (self.meter, "zeros")]
        self.fake = _FakeC()
        self.aud = SA.Auditor(SPEC, self.fake, params, initial, values=False)
        self.C = SA._Proxy(self.fake, self.aud)
        self.step, self.accum = 0, 0

    def v(self, arena, name):
        a, b = self.off[name]
        return arena[a:b]

    def w(self, layer):
        return self.v(self.w16, layer + ".weight")

    def b(self, layer):
        return self.v(self.p32, layer + ".bias")

    def g(self, name):
        return self.v(self.g32, name)

    # ------------------------------------------------------------------------------------------
    def _input(self, batch):
        imgs, prm, lab = batch
        j = self.slot
        self.slot ^= 1
        self.src[j].copy_(imgs)
        self.prm[j].copy_(prm)
        self.lab[j].copy_(lab)
        src = self.src[j ^ 1] if self.defect == "input_slot" else self.src[j]
        self.C.augment(src, self.prm[j], self.x, 8, 8, HW, HW, 0, 4, [0.5] * 3, [0.25] * 3)
        self.aud.flush_labels("input", None)
        return j

    def _forward(self):
        C = self.C
        C.conv0_fprop(self.x, self.w("features.0"), self.b("features.0"), self.acts[0])
        self.aud.mark("fwd features.0")
        x = self.acts[0]
        for i, c in enumerate(SPEC.convs[1:], start=1):
            if c.pool_after:
                C.conv_fprop_pool(x, self.w(c.name), self.b(c.name), self.pools[i], self.masks[i], 0)
                x = self.pools[i]
            else:
                C.conv_fprop(x, self.w(c.name), self.b(c.name), self.acts[i], True, 0)
                x = self.acts[i]
                if self.defect == "unrecorded_write":
                    x.view(-1)[0] += 1
            self.aud.mark("fwd " + c.name)
        self.feat = x.reshape(B, -1)
        C.gemm(self.w("classifier.0"), False, self.feat, False, 16, B, 64, self.fc_acc, 16, C.EPI_F32_ATOMIC_T, None,
               1.0, 1, 0)
        C.fc_bias_act(self.fc_acc, self.b("classifier.0"), self.fc_y, None, B, 16, True, 0.5, 7, self.step, True)
        self.aud.flush_labels("fwd", None)

    def _head(self, j, train):
        C = self.C
        if train:
            args = (self.fc_y, self.w("classifier.3"), self.b("classifier.3"), self.lab[j], self.logits, self.fc_dz[1],
                    8, self.g("classifier.3.weight"), self.g("classifier.3.bias"), self.fc_dz[0], 2.0, True,
                    self.meter, self.loss, None)
            C.head_ce(*(args + ((True,) if self.accum else ())))
        else:
            C.head_ce(self.fc_y, self.w("classifier.3"), self.b("classifier.3"), self.lab[j], self.logits, None, 0,
                      None, None, None, 1.0, False, self.meter, self.loss, None)
        self.aud.flush_labels("loss", None)

    def _opt(self, name):
        if not self.update:
            return
        self.aud.mark("opt start")
        a, b = self.off[name]
        g = self.g32[a:b]
        self.C.adam(self.p32[a:b], self.m32[a:b], self.v32[a:b], g, None, self.w16[a:b], 1e-3, 0.9, 0.999, 1e-8,
                    0.0, self.step, 1.0 / (self.accum + 1), g)
        self.aud.mark("opt end")

    def _backward(self):
        C = self.C
        self._opt("classifier.3.bias")
        self._opt("classifier.3.weight")
        self.aud.mark("bwd classifier.3")
        dz = self.fc_dz[0]
        C.bias_grad(dz, self.g("classifier.0.bias"), B, 16, 16, 1.0)
        self._opt("classifier.0.bias")
        C.gemm(dz, True, self.feat, True, 16, 64, B, self.g("classifier.0.weight"), 64,
               C.EPI_F32_ATOMIC if self.accum else C.EPI_F32_STORE, None, 1.0, 1, 0)
        C.gemm(self.w("classifier.0"), True, dz, False, 64, B, 16, self.fc_dacc, 64, C.EPI_F32_STORE_T, None, 1.0, 1, 0)
        self._opt("classifier.0.weight")
        C.fc_grad_act(self.fc_dacc, None, self.dfeat.view(B, -1), B, 64, False, 0.0, True)
        self.aud.mark("bwd classifier.0")
        g, pp, convs = self.dfeat, 0, SPEC.convs
        for i in range(len(convs) - 1, -1, -1):
            c = convs[i]
            y = self.acts[i]
            if c.pool_after:
                dz = self.dbuf[pp][:y.numel()].view_as(y)
                C.unpool2x2(g, self.masks[i], dz, self.g(c.name + ".bias"))
                if i == 3 and self.defect == "bias_twice":
                    C.bias_grad(dz, self.g(c.name + ".bias"), dz.numel() // c.cout, c.cout, c.cout, 1.0)
                pp ^= 1
            else:
                dz = g
            self._opt(c.name + ".bias")
            if i == 0:
                C.conv0_wgrad(dz, self.x, self.g(c.name + ".weight"))
                self._opt(c.name + ".weight")
                self.aud.mark("bwd " + c.name)
                break
            prev = convs[i - 1]
            x_in = self.pools[i - 1] if prev.pool_after else self.acts[i - 1]
            wgrad_dz, wgrad_x, dw = dz, x_in, self.g(c.name + ".weight")
            if i == 2 and self.defect == "ping_pong":
                wgrad_dz = self.dbuf[pp][:dz.numel()].view_as(dz)
            if i == 2 and self.defect == "stale_activation":
                wgrad_x = self.acts[i - 1]
            if i == 2 and self.defect == "wrong_slot":
                dw = self.g(convs[i + 1].name + ".weight")
            C.conv_wgrad(wgrad_dz, wgrad_x, dw, 1.0, 0, 0)
            dx = self.dbuf[pp ^ 1 if self.defect == "alias" else pp][:x_in.numel()].view_as(x_in)
            fuse = not prev.pool_after
            if self.defect == "early_update":
                self._opt(c.name + ".weight")
            C.conv_dgrad(dz, self.w(c.name), x_in if fuse else None, dx, self.g(prev.name + ".bias") if fuse else None,
                         0)
            if self.defect != "early_update":
                self._opt(c.name + ".weight")
            self.aud.mark("bwd " + c.name)
            pp ^= 1
            g = dx

    # ------------------------------------------------------------------------------------------
    def train_step(self, batch, update=True):
        self.step += 1
        self.update = update
        self.aud.begin_step("train", images=batch[0], params=batch[1], labels=batch[2], update=update)
        j = self._input(batch)
        self._forward()
        self._head(j, True)
        self.aud.mark("loss")
        self._backward()
        self.aud.end_step()
        self.accum = 0 if update else self.accum + 1

    def eval_step(self, batch):
        self.aud.begin_step("eval", images=batch[0], params=batch[1], labels=batch[2])
        j = self._input(batch)
        self._forward()
        self._head(j, False)
        self.aud.end_step()


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 256, (B, 8, 8, 3), generator=g, dtype=torch.uint8), torch.rand(B, 8, generator=g),
            torch.randint(0, 3, (B,), generator=g))


def _run(defect=None):
    eng = _MiniEngine(defect)
    eng.train_step(_batch(1))
    eng.train_step(_batch(2))
    eng.eval_step(_batch(3))
    eng.train_step(_batch(4), update=False)
    eng.train_step(_batch(5), update=True)
    return eng.aud


def test_clean_sequence_passes():
    aud = _run()
    assert aud.counts["conv_fprop_pool"] == 2 * 5 and aud.counts["adam"] == 3 * len(SPEC.param_names)
    assert aud.links > 200


DEFECTS = {
    "ping_pong": r"conv_wgrad \(bwd features\.5\): argument dz .* expected producer bwd features\.7 "
                 r"conv_dgrad\.dx of this step, found step \d+ #\d+ bwd features\.7 unpool2x2\.dz",
    "stale_activation": r"conv_wgrad \(bwd features\.5\): argument x .* expected producer fwd features\.2 "
                        r"conv_fprop_pool\.pooled .* found nothing \(never written\)",
    "unrecorded_write": r"conv_fprop_pool \(fwd features\.7\): argument x changed after its producer .* fwd features\.5 "
                        r"conv_fprop\.y wrote it .*: a write the audit did not see",
    "alias": r"conv_dgrad \(bwd features\.7\): written argument dx overlaps argument dz",
    "early_update": r"conv_dgrad \(bwd features\.7\): argument w .* expected producer features\.7\.weight as "
                    r"initialised, found step 0 #\d+ opt adam\.shadow",
    "wrong_slot": r"gradient slot of features\.5\.weight written by 0 launches",
    "bias_twice": r"gradient slot of features\.7\.bias written by 2 launches \(#\d+ bwd features\.7 unpool2x2\.colsum, "
                  r"#\d+ bwd features\.7 bias_grad\.db\)",
    "input_slot": r"step 0 launch #\d+ augment \(input -\): argument src is not the images of the batch",
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_planted_defect_is_reported(defect):
    with pytest.raises(SA.AuditError, match=DEFECTS[defect]):
        _run(defect)
