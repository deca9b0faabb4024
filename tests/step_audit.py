"""Audit every kernel launch of real training steps on the engine's own tensors.

The kernel tests and the launch replay (launch_replay.py) check each kernel on fresh operands.  This
module checks the glue between the kernels: whether each launch of ``NativeEngine`` gets the right
buffers, in the right order, holding what the previous launch left there.  ``audit_engine`` swaps
``ops._C`` for a proxy, the way ``launch_replay._Recorder`` does; the engine runs unmodified.  For
every call of a kernel in ``launch_replay.RECORDED`` the proxy synchronises the device, snapshots
every tensor argument (the exact view passed), makes the call and synchronises again.  Launches are
attributed to a layer by wrapping the instance's ``_mark`` ("fwd features.12", "bwd classifier.0",
"opt3 start" ...) and ``_stage_input`` / ``_forward`` / ``_loss`` (the head and the input have no
marks); a forward launch, or one without a layer mark, takes the layer whose parameters it reads.

Because every launch is followed by a device synchronise, the side streams (optimizer, input
copies) are serialised in the order the engine enqueues work.  The audit therefore checks enqueue
order, not the cross-stream event waits: a missing ``wait_event`` is invisible to it.

Three checks per launch:

(a) values: ``launch_replay.verify`` against the float64 reference, evaluated on the snapshots
    taken before the launch (kernel_check's bounds, gauss mode; accumulation targets as before plus
    the contribution);
(b) arguments: no written argument overlaps another argument of the same launch, except the
    optimizer clearing the gradient it reads (``zero`` is ``g32``);
(c) links: every argument the launch reads (read-only, accumulated or updated) holds, bit for bit,
    what its prescribed producer left in that memory.  The producers come from a dataflow table
    written here from the ``VGGSpec`` (``_expect``), with both routes allowed per layer (fused or
    separate pool, fused head or GEMM + fc_bias_act + cross_entropy).  Writes the audit cannot
    intercept are named in ``EXTERNAL`` and ``initial`` buffers, each with its reason; any other
    change of a region between its producer and a consumer fails.  Each parameter's gradient slot
    must receive exactly one weight- or bias-gradient contribution per micro-batch, from its
    prescribed kernel, and nothing else.

The byte-level model covers each argument's contiguous extent; the engine passes contiguous views
only, and the audit refuses any other.  ``Auditor`` itself is independent of the engine and of the
GPU, so test_step_audit_cpu.py drives it with a scripted fake extension on CPU tensors.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional

import torch

import kernel_check as KC
import launch_replay as LR

READ, STORE, ACCUM, UPDATE = LR.READ, LR.STORE, LR.ACCUM, LR.UPDATE

# Arguments written outside any recorded launch: (kernel, argument) -> (what the batch the caller
# passed in says it must equal, why the audit cannot see the write).
EXTERNAL = {
    ("augment", "src"): ("images", "H2D copy of the caller's uint8 images on the copy stream"),
    ("augment", "params"): ("params", "H2D copy of the caller's crop parameters on the copy stream"),
    ("nchw_to_nhwc", "x"): ("images", "the caller's float images, moved to the device by torch"),
    ("cross_entropy", "target"): ("labels", "copy of the caller's labels (copy stream or torch copy_)"),
    ("head_ce", "target"): ("labels", "copy of the caller's labels (copy stream or torch copy_)"),
    ("cross_entropy", "class_weights"): ("class_weights", "set by the caller through set_class_weights"),
    ("head_ce", "class_weights"): ("class_weights", "set by the caller through set_class_weights"),
}


class AuditError(AssertionError):
    pass


class _Deferred(Exception):
    """A failed check of a launch whose layer is not known yet: raised as an AuditError once the
    next mark names it."""

    def __init__(self, launch, msg):
        super().__init__(msg)
        self.launch, self.msg = launch, msg


def _desc(d):
    phase, layer, kind, key = d
    return "%s %s%s.%s" % (phase, (layer + " ") if layer else "", kind, key)


class _Write:
    """What one launch left in one region: the bytes, for the links of later readers."""
    __slots__ = ("launch", "key", "a0", "bytes", "what")

    def __init__(self, launch, key, a0, data, what=None):
        self.launch, self.key, self.a0, self.bytes, self.what = launch, key, a0, data, what

    def desc(self):
        if self.launch is None:
            return self.what
        L = self.launch
        return "step %d #%d %s" % (L.step, L.seq, _desc(L.desc(self.key)))


class _Launch:
    __slots__ = ("seq", "step", "name", "kind", "phase", "layer", "args", "sc", "roles", "reads", "writes")

    def __init__(self, seq, step, name, kind):
        self.seq, self.step, self.name, self.kind = seq, step, name, kind
        self.phase = self.layer = None
        self.reads, self.writes = {}, {}

    def desc(self, key):
        return (self.phase, self.layer, self.kind, key)

    def title(self):
        return "step %d launch #%d %s (%s %s)" % (self.step, self.seq, self.kind, self.phase, self.layer or "-")


def _bytes(t):
    if not t.is_contiguous():
        raise AuditError("non-contiguous argument %s %s: the audit models contiguous extents" %
                         (tuple(t.shape), tuple(t.stride())))
    return t.reshape(-1).view(torch.uint8)


def _extent(t):
    """(storage, first byte, one past the last byte) of a contiguous view."""
    esz = t.element_size()
    return t.untyped_storage().data_ptr(), t.storage_offset() * esz, (t.storage_offset() + t.numel()) * esz


class Auditor:
    """The bookkeeping of the audit, independent of the engine.

    ``spec``: the VGGSpec the dataflow table is written from.  ``C``: the extension (or a fake one)
    whose kernels are called.  ``params``: parameter name -> (the view launches read, the gradient
    slot).  ``initial``: (tensor, reason) regions whose content before the audit counts as written.
    ``values``: run check (a) (needs the GPU references)."""

    def __init__(self, spec, C, params: Dict[str, tuple], initial=(), values: bool = True, sms: int = 0):
        self.spec, self.C, self.values, self.sms = spec, C, values, sms
        self.params = params
        self.mem: Dict[int, list] = {}                  # storage -> sorted [lo, hi, _Write]
        self.seq = 0
        self.step = -1
        self.launches: List[_Launch] = []                # of the current step
        self.pending: List[_Launch] = []
        self.bracket = None
        self.failed: Optional[_Deferred] = None
        self.expect_batch: dict = {}
        self.counts: Dict[str, int] = {}
        self.links = 0
        self.update = True                               # the current training step ends with an update
        self.last_update_step = None                     # step whose optimizer wrote the current weights
        self.group: List[int] = []                       # steps of the open accumulation group
        self.contrib: Dict[int, Dict[str, list]] = {}    # step -> parameter -> [(launch, key, exact slot)]
        self.kind_of_step: Dict[int, str] = {}
        self.convs = [c.name for c in spec.convs]
        self.fcs = [f.name for f in spec.fcs]
        self._slot = {}
        for name, (view, grad) in params.items():
            self._slot[name] = (_extent(view), _extent(grad))
        for t, why in initial:
            self._write(None, "initial", t, what="initial " + why)

    # ------------------------------------------------------------------------------ memory model
    def _write(self, launch, key, t, what=None):
        s, a, b = _extent(t)
        if b == a:
            return
        rec = _Write(launch, key, a, _bytes(t).clone(), what)
        ivs = self.mem.setdefault(s, [])
        out = []
        for lo, hi, w in ivs:
            if hi <= a or lo >= b:
                out.append([lo, hi, w])
                continue
            if lo < a:
                out.append([lo, a, w])
            if hi > b:
                out.append([b, hi, w])
        out.append([a, b, rec])
        out.sort(key=lambda iv: iv[0])
        self.mem[s] = out

    def _cover(self, s, a, b):
        """[(lo, hi, _Write or None for never written)] over [a, b)."""
        pieces, pos = [], a
        for lo, hi, w in self.mem.get(s, ()):
            if hi <= a or lo >= b:
                continue
            if lo > pos:
                pieces.append((pos, lo, None))
            pieces.append((max(lo, a), min(hi, b), w))
            pos = min(hi, b)
        if pos < b:
            pieces.append((pos, b, None))
        return pieces

    # ----------------------------------------------------------------------------- step framing
    def begin_step(self, kind: str, images=None, params=None, labels=None, class_weights=None,
                   update: bool = True):
        """kind: "train" or "eval"; the rest is the batch the caller passed in."""
        self.flush_labels("?", None)
        self.step += 1
        self.kind_of_step[self.step] = kind
        self.update = update
        self.expect_batch = {"images": images, "params": params, "labels": labels, "class_weights": class_weights}
        self.launches = []
        if kind == "train":
            self.group.append(self.step)
            self.contrib[self.step] = {}

    def end_step(self):
        self.flush_labels("?", None)
        for L in self.launches:
            if L.phase == "?":
                raise AuditError("%s: no layer mark followed the launch" % L.title())
        if self.kind_of_step[self.step] == "train":
            self._check_contributions()
        for L in self.launches:
            self._links(L)
        if self.kind_of_step[self.step] == "train":
            if self.update:
                self.last_update_step = self.step
                self.group = []
        self.launches = []

    # ------------------------------------------------------------------------------ attribution
    def mark(self, name: str):
        if name.startswith("fwd ") or name.startswith("bwd "):
            self.flush_labels(name[:3], name[4:])
        elif name.startswith("opt") and name.endswith(" start"):
            self.bracket = ("opt", None)
        elif name.startswith("opt") and name.endswith(" end"):
            self.bracket = None
        elif name == "input":
            self.flush_labels("input", None)
        elif name == "loss":
            self.flush_labels("loss", None)

    def flush_labels(self, phase, layer):
        for L in self.pending:
            L.phase = phase
            # the forward marks only some layers (conv0 has none): a forward launch belongs to the layer
            # whose parameters it reads
            by = self._layer_by_params(L)
            L.layer = by if by is not None and (layer is None or phase == "fwd") else layer
        self.pending = []
        self._raise_failed()

    def _raise_failed(self):
        if self.failed is not None and self.failed.launch.phase is not None:
            raise AuditError("%s: %s" % (self.failed.launch.title(), self.failed.msg))

    def _layer_by_params(self, L):
        ext = {_extent(t) for t in L.args.values() if isinstance(t, torch.Tensor)}
        for name, (view, _) in self._slot.items():
            if view in ext:
                return name.rsplit(".", 1)[0]
        return None

    # ---------------------------------------------------------------------------------- launches
    def _role(self, name, key, sc):
        if name == "gemm" and key == "out":
            return ACCUM if sc["code"] in (self.C.EPI_F32_ATOMIC, self.C.EPI_F32_ATOMIC_T) else STORE
        if key == "acc":
            return UPDATE if sc["clear"] else READ
        if name == "head_ce" and key == "dW":
            return ACCUM if sc.get("accumulate") else STORE
        if name in ("adam", "sgd") and key == "g32" and sc.get("_zero_is_g32"):
            return UPDATE
        return LR.CONTRACT[name][key]

    def launch(self, name, args, fn):
        """Audit one call ``fn(*args)`` of kernel ``name``.  After a failed check no kernel runs; the
        failure is raised as soon as the launch's layer is known."""
        if self.failed is not None:
            return
        try:
            self._launch(name, args, fn)
        except _Deferred as d:
            self.failed = d
            self._raise_failed()

    def _launch(self, name, args, fn):
        tensors, sc = LR.split_args(name, args)
        kind = name
        if name == "gemm":
            kind = {(False, False): "gemm.fwd", (True, True): "gemm.wgrad", (True, False): "gemm.dgrad"}.get(
                (bool(sc["a_mn"]), bool(sc["b_mn"])), "gemm")
        if name in ("adam", "sgd"):
            z, g = tensors.get("zero"), tensors.get("g32")
            sc["_zero_is_g32"] = z is not None and g is not None and _extent(z) == _extent(g)
        L = _Launch(self.seq, self.step, name, kind)
        self.seq += 1
        L.args, L.sc = tensors, sc
        L.roles = {k: self._role(name, k, sc) for k, t in tensors.items() if t is not None}
        if self.bracket is not None:
            L.phase, L.layer = self.bracket
        else:
            L.phase = None
            self.pending.append(L)
        self.launches.append(L)
        self.counts[name] = self.counts.get(name, 0) + 1
        sync = torch.cuda.synchronize if any(t.is_cuda for t in L.args.values() if t is not None) else (lambda: None)
        sync()
        self._overlap(L)
        before = {k: (None if t is None else t.clone()) for k, t in tensors.items()}
        for k, role in L.roles.items():
            if role != STORE:
                L.reads[k] = self._read(L, k, before[k])
        fn(*args)
        sync()
        if self.values:
            try:
                LR.verify(name, before, tensors, sc, self.sms, exact=False, what=name)
            except AssertionError as e:
                raise _Deferred(L, "value check failed: %s" % e)
        for k, role in L.roles.items():
            if role != READ:
                self._write(L, k, tensors[k])
                L.writes[k] = _extent(tensors[k])
        self._contribute(L)

    def _overlap(self, L):
        ext = {k: _extent(t) for k, t in L.args.items() if t is not None}
        for k, role in L.roles.items():
            if role == READ:
                continue
            s, a, b = ext[k]
            for k2, (s2, a2, b2) in ext.items():
                if k2 == k or s2 != s or b2 <= a or a2 >= b:
                    continue
                if L.name in ("adam", "sgd") and {k, k2} == {"zero", "g32"} and (a, b) == (a2, b2):
                    continue
                raise _Deferred(L, "written argument %s overlaps argument %s in memory (bytes [%d, %d) and "
                                "[%d, %d))" % (k, k2, a, b, a2, b2))

    def _read(self, L, key, snap):
        """Who wrote what ``key`` reads; the bytes must be what they left."""
        ext = (L.name, key)
        if ext in EXTERNAL:
            field, why = EXTERNAL[ext]
            want = self.expect_batch.get(field)
            if want is None:
                raise _Deferred(L, "argument %s (%s) but the caller passed no %s" % (key, why, field))
            want = torch.as_tensor(want).to(snap.device, snap.dtype).reshape(snap.shape)
            if not torch.equal(snap, want):
                raise _Deferred(L, "argument %s is not the %s of the batch the caller passed in (%s)" %
                                (key, field, why))
            return [("external", why)]
        s, a, b = _extent(L.args[key])
        cur = _bytes(snap)
        found = []
        for lo, hi, w in self._cover(s, a, b):
            if w is not None and not torch.equal(cur[lo - a:hi - a], w.bytes[lo - w.a0:hi - w.a0]):
                raise _Deferred(L, "argument %s changed after its producer %s wrote it (bytes [%d, %d)): a write "
                                "the audit did not see" % (key, w.desc(), lo, hi))
            found.append((lo, hi, w))
        return found

    # ----------------------------------------------------------------------- gradient contributions
    def _contribute(self, L):
        if self.kind_of_step.get(L.step) != "train" or L.phase == "opt" or L.name in ("adam", "sgd"):
            return
        for k, (s, a, b) in L.writes.items():
            for name, (_, (gs, ga, gb)) in self._slot.items():
                if gs == s and a < gb and b > ga:
                    self.contrib[L.step].setdefault(name, []).append((L, k, (a, b) == (ga, gb)))

    def _prescribed_grad(self, name):
        """(phase, layer, kind, key) of the launches that may write parameter ``name``'s gradient."""
        layer, what = name.rsplit(".", 1)
        sp = self.spec
        if layer in self.convs:
            i = self.convs.index(layer)
            c = sp.convs[i]
            if what == "weight":
                return [("bwd", layer, "conv0_wgrad" if i == 0 else "conv_wgrad", "dw0" if i == 0 else "dw")]
            out = [("bwd", layer, "bias_grad", "db")]
            if c.pool_after:
                out += [("bwd", layer, "unpool2x2", "colsum"), ("bwd", layer, "maxpool_relu_bwd", "colsum")]
            elif i + 1 < len(sp.convs):
                out.append(("bwd", self.convs[i + 1], "conv_dgrad", "colsum"))
            return out
        last = layer == self.fcs[-1]
        if what == "weight":
            return [("bwd", layer, "gemm.wgrad", "out")] + ([("loss", layer, "head_ce", "dW")] if last else [])
        return [("bwd", layer, "bias_grad", "db")] + ([("loss", layer, "head_ce", "db")] if last else [])

    def _check_contributions(self):
        got = self.contrib[self.step]
        for name in self.params:
            allowed = self._prescribed_grad(name)
            c = got.get(name, [])
            descs = ["#%d %s" % (L.seq, _desc(L.desc(k))) for L, k, _ in c]
            if len(c) != 1:
                raise AuditError("step %d: gradient slot of %s written by %d launches (%s); expected exactly one of "
                                 "%s" % (self.step, name, len(c), ", ".join(descs) or "none",
                                         " / ".join(_desc(d) for d in allowed)))
            L, k, exact = c[0]
            if L.desc(k) not in allowed or not exact:
                raise AuditError("step %d: gradient slot of %s written by %s%s; expected %s" % (
                    self.step, name, descs[0], "" if exact else " (not exactly the slot)",
                    " / ".join(_desc(d) for d in allowed)))
        self.links += len(self.params)

    # -------------------------------------------------------------------------------------- links
    def _param_of(self, L, key):
        """The parameter whose read view is exactly this argument, if any."""
        e = _extent(L.args[key])
        for name, (view, _) in self._slot.items():
            if view == e:
                return name
        return None

    def _expect(self, L, key):
        """The prescribed producer of what launch L reads through ``key``: ("param", name),
        ("grad", None), ("state", [descs]) (any earlier step, or the initial content) or
        ("step", [descs]) (this step)."""
        k, lay = L.kind, L.layer
        sp, convs, fcs = self.spec, self.convs, self.fcs
        P = lambda what: ("param", "%s.%s" % (lay, what))          # noqa: E731

        def out_of(i):                       # what conv layer i hands to layer i + 1
            c = sp.convs[i]
            if c.pool_after:
                return [("fwd", convs[i], "conv_fprop_pool", "pooled"), ("fwd", convs[i], "maxpool_fwd", "y")]
            return [act_of(i)]

        def act_of(i):                       # conv layer i's stored post-ReLU activation
            return ("fwd", convs[0], "conv0_fprop", "y") if i == 0 else ("fwd", convs[i], "conv_fprop", "y")

        inp = [("input", None, "augment", "out"), ("input", None, "nchw_to_nhwc", "y")]
        feat = out_of(len(convs) - 1) + [("fwd", None, "avgpool_fwd", "y")]

        def fc_in(j):                        # the input of FC layer j
            return feat if j == 0 else [("fwd", fcs[j - 1], "fc_bias_act", "y")]

        def fc_dz(j):                        # the gradient wrt FC layer j's output, as its backward reads it
            if j == len(fcs) - 1:
                return [("loss", None, "cross_entropy", "dlogits"), ("loss", fcs[j], "head_ce", "dlogits")]
            return [("bwd", fcs[j + 1], "fc_grad_act", "dz"), ("loss", fcs[j + 1], "head_ce", "dh")]

        def opener(i):                       # what opened conv layer i's backward (its dz)
            if sp.convs[i].pool_after:
                return [("bwd", convs[i], "unpool2x2", "dz"), ("bwd", convs[i], "maxpool_relu_bwd", "dz")]
            return [("bwd", convs[i + 1], "conv_dgrad", "dx")]

        def dpool(i):                        # the gradient wrt pooled layer i's output
            if i == len(convs) - 1:
                return [("bwd", fcs[0], "fc_grad_act", "dz"), ("bwd", convs[i], "avgpool_bwd", "dx")]
            return [("bwd", convs[i + 1], "conv_dgrad", "dx")]

        if L.name in ("adam", "sgd"):
            if key in ("g32", "zero"):
                return ("grad", None)
            return ("state", [("opt", None, L.name, key)])
        if L.name in ("cross_entropy", "head_ce") and key == "meter":
            return ("state", [("loss", None, "cross_entropy", "meter"), ("loss", fcs[-1], "head_ce", "meter")])
        if L.roles[key] in (ACCUM, UPDATE) and self._grad_param(L, key):
            return ("grad", None)
        ci = convs.index(lay) if lay in convs else None
        fi = fcs.index(lay) if lay in fcs else None
        table = {
            ("conv0_fprop", "x4"): ("step", inp), ("conv0_fprop", "w0"): P("weight"),
            ("conv0_fprop", "bias"): P("bias"),
            ("conv_fprop", "w"): P("weight"), ("conv_fprop", "bias"): P("bias"),
            ("conv_fprop_pool", "w"): P("weight"), ("conv_fprop_pool", "bias"): P("bias"),
            ("conv_dgrad", "w"): P("weight"), ("gemm.fwd", "A"): P("weight"), ("gemm.dgrad", "A"): P("weight"),
            ("fc_bias_act", "bias"): P("bias"), ("head_ce", "W"): P("weight"), ("head_ce", "bias"): P("bias"),
            ("maxpool_fwd", "x"): ("step", [act_of(ci)] if ci is not None else []),
            ("avgpool_fwd", "x"): ("step", out_of(len(convs) - 1)),
            ("avgpool_bwd", "dy"): ("step", [("bwd", fcs[0], "fc_grad_act", "dz")]),
            ("cross_entropy", "logits"): ("step", [("fwd", fcs[-1], "fc_bias_act", "y_f32")]),
            ("head_ce", "h"): ("step", fc_in(len(fcs) - 1)),
        }
        if ci is not None:
            x_in = inp if ci == 0 else out_of(ci - 1)
            table.update({
                ("conv_fprop", "x"): ("step", x_in), ("conv_fprop_pool", "x"): ("step", x_in),
                ("unpool2x2", "dp"): ("step", dpool(ci)), ("maxpool_relu_bwd", "dp"): ("step", dpool(ci)),
                ("unpool2x2", "mask"): ("step", [("fwd", lay, "conv_fprop_pool", "mask")]),
                ("maxpool_relu_bwd", "y"): ("step", [act_of(ci)]),
                ("conv_wgrad", "dz"): ("step", opener(ci)), ("conv_wgrad", "x"): ("step", x_in),
                ("conv_dgrad", "dz"): ("step", opener(ci)),
                ("conv0_wgrad", "dz"): ("step", opener(0)), ("conv0_wgrad", "x4"): ("step", inp),
                ("bias_grad", "dz"): ("step", opener(ci)),
            })
            if ci > 0:
                table[("conv_dgrad", "mask_src")] = ("step", [act_of(ci - 1)])
        if fi is not None:
            table.update({
                ("gemm.fwd", "B"): ("step", fc_in(fi)),
                ("gemm.fwd", "out"): ("state", [("fwd", lay, "fc_bias_act", "acc")]),
                ("fc_bias_act", "acc"): ("step", [("fwd", lay, "gemm.fwd", "out")]),
                ("bias_grad", "dz"): ("step", fc_dz(fi)),
                ("gemm.wgrad", "A"): ("step", fc_dz(fi)), ("gemm.wgrad", "B"): ("step", fc_in(fi)),
                ("gemm.dgrad", "B"): ("step", fc_dz(fi)),
                ("gemm.dgrad", "out"): ("state", [("bwd", lay, "fc_grad_act", "acc")]),
                ("fc_grad_act", "acc"): ("step", [("bwd", lay, "gemm.dgrad", "out")]),
                ("fc_grad_act", "act"): ("step", fc_in(fi)),
            })
        if (k, key) not in table:
            raise AuditError("%s: no prescribed producer for argument %s" % (L.title(), key))
        return table[(k, key)]

    def _grad_param(self, L, key):
        s, a, b = _extent(L.args[key])
        for name, (_, (gs, ga, gb)) in self._slot.items():
            if gs == s and a < gb and b > ga:
                return name
        return None

    def _links(self, L):
        for key, found in L.reads.items():
            if found and found[0][0] == "external":
                self.links += 1
                continue
            how, want = self._expect(L, key)
            if how == "param":
                self._link_param(L, key, want, found)
            elif how == "grad":
                self._link_grad(L, key, found)
            else:
                for lo, hi, w in found:
                    ok = w is not None and (
                        (w.launch is None and how == "state") or
                        (w.launch is not None and w.launch.desc(w.key) in want and
                         (how == "state" or w.launch.step == L.step)))
                    if not ok:
                        self._fail(L, key, lo, hi, w, " / ".join(_desc(d) for d in want) +
                                   (" of this step" if how == "step" else " (or the initial content)"))
            self.links += 1

    def _fail(self, L, key, lo, hi, w, expected):
        found = "nothing (never written)" if w is None else w.desc()
        raise AuditError("%s: argument %s (bytes [%d, %d)) expected producer %s, found %s" %
                         (L.title(), key, lo, hi, expected, found))

    def _link_param(self, L, key, name, found):
        got = self._param_of(L, key)
        if got != name:
            raise AuditError("%s: argument %s reads %s, expected the parameter %s" %
                             (L.title(), key, got or "a region that is no parameter", name))
        upd = self.last_update_step
        for lo, hi, w in found:
            if upd is None:
                ok = w is not None and w.launch is None
            else:
                ok = w is not None and w.launch is not None and w.launch.step == upd and w.launch.phase == "opt"
            if not ok:
                self._fail(L, key, lo, hi, w, "%s as the optimizer of step %s left it" % (name, upd) if upd is not None
                           else "%s as initialised" % name)

    def _link_grad(self, L, key, found):
        """Gradient slots: the first micro-batch of a group reads what the optimizer cleared (or the
        initial zeros), later ones what the previous micro-batch's contributor left; the optimizer
        reads what this micro-batch's contributors left."""
        for lo, hi, w in found:
            name = None
            s = _extent(L.args[key])[0]
            for n, (_, (gs, ga, gb)) in self._slot.items():
                if gs == s and lo < gb and hi > ga:
                    name = n
            if L.name in ("adam", "sgd"):
                if name is None:
                    continue                 # alignment padding between slots
                allowed = self._prescribed_grad(name)
                ok = w is not None and w.launch is not None and w.launch.step == L.step and \
                    w.launch.desc(w.key) in allowed
                expected = "the gradient of %s from %s of this step" % (name, " / ".join(_desc(d) for d in allowed))
            elif len(self.group) > 1 and L.step == self.group[-1]:
                prev = self.group[-2]
                allowed = self._prescribed_grad(name) if name else []
                ok = w is not None and w.launch is not None and w.launch.step == prev and \
                    w.launch.desc(w.key) in allowed
                expected = "the gradient of %s from step %d (the group's previous micro-batch)" % (name, prev)
            else:
                ok = w is not None and (w.launch is None or w.launch.phase == "opt")
                expected = "the gradient slot of %s as the optimizer cleared it (or the initial zeros)" % name
            if not ok:
                self._fail(L, key, lo, hi, w, expected)


class _Proxy:
    """Stands in for the extension module: audits the recorded kernels, forwards everything else."""

    def __init__(self, real, auditor):
        self._real, self._aud = real, auditor

    def __getattr__(self, name):
        attr = getattr(self._real, name)
        if name not in LR.RECORDED:
            return attr

        def call(*args):
            return self._aud.launch(name, args, attr)
        return call


def engine_auditor(eng, values=True):
    """An Auditor over a NativeEngine's parameter views, gradient slots and initial buffers."""
    params = {}
    for name in eng.spec.param_names:
        arena = eng.w16 if name.endswith(".weight") else eng.p32
        params[name] = (eng._view(arena, name), eng._view(eng.g32, name))
    initial = [(eng.p32, "parameters (import_state)"), (eng.w16, "bf16 weight shadow (import_state)"),
               (eng.m32, "optimizer state (zeros)"), (eng.g32, "gradient arena (zeros)"),
               (eng.scratch_meter, "loss meter (zeros)")]
    if eng.v32 is not None:
        initial.append((eng.v32, "optimizer state (zeros)"))
    initial += [(t, "FC forward accumulator (zeros)") for t in eng.fc_acc]
    initial += [(t, "FC dgrad accumulator (zeros)") for t in eng.fc_dacc]
    from distributed_vgg_f_b200 import ops

    return Auditor(eng.spec, ops.require(), params, initial, values=values, sms=KC.sm_count() if values else 0)


def _batch_fields(batch):
    from distributed_vgg_f_b200.data.loader import FusedBatch

    if isinstance(batch, FusedBatch):
        return {"images": batch.images_u8, "params": batch.params, "labels": batch.labels}
    x, y = batch
    return {"images": x, "labels": y}


@contextlib.contextmanager
def audit_engine(eng, values=True):
    """Audit every launch of ``eng.train_step`` / ``eng.eval_step`` inside the block.  Yields the
    Auditor; the engine is restored when the block ends."""
    from distributed_vgg_f_b200 import ops

    aud = engine_auditor(eng, values=values)
    real = ops.require()
    orig = {k: getattr(eng, k) for k in ("_mark", "_stage_input", "_forward", "_loss", "train_step", "eval_step")}

    def mark(name, lane="compute"):
        aud.mark(name)
        return orig["_mark"](name, lane)

    def stage(batch):
        b = orig["_stage_input"](batch)
        aud.flush_labels("input", None)
        return b

    def forward(b, train):
        orig["_forward"](b, train)
        aud.flush_labels("fwd", None)

    def loss(b, train):
        orig["_loss"](b, train)
        aud.flush_labels("loss", None)

    def train_step(batch, update=True):
        aud.begin_step("train", class_weights=eng.class_weights, update=update, **_batch_fields(batch))
        out = orig["train_step"](batch, update=update)
        aud.end_step()
        return out

    def eval_step(batch):
        aud.begin_step("eval", **_batch_fields(batch))
        out = orig["eval_step"](batch)
        aud.end_step()
        return out

    eng._mark, eng._stage_input, eng._forward, eng._loss = mark, stage, forward, loss
    eng.train_step, eng.eval_step = train_step, eval_step
    ops._C = _Proxy(real, aud)
    try:
        yield aud
    finally:
        ops._C = real
        for k in orig:
            delattr(eng, k)
