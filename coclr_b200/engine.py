"""Host-side executor of one encoder (S3D backbone + MoCo projection head) on the sm_90a kernels.

The reference runs `encoder_q(x1)` / `encoder_k(x2)` (model/pretrain.py:153,165) as ~250 PyTorch
module calls; here an encoder pass is a pre-built list of C-ABI kernel launches over pre-allocated
channels-last buffers:

  clip pack -> [conv (+BN statistics in the epilogue) -> BN finalize]* with BN-apply/ReLU folded into
  the next operand load, max-pools, concat-by-slice -> avg-pool -> 2 head convs -> L2-normalise

and the backward pass is the mirrored list (BN backward in place, dgrad, wgrad into one flat
gradient buffer).  Parameters live in ONE flat fp32 buffer per encoder (nn.Parameters are views), so
EMA / Adam / all-reduce are single launches over it.
"""
import ctypes as C
from collections import namedtuple

import torch

from . import lib as L
from . import ops
from .s3d_spec import s3d_stages, S3D_FEATURE_SIZE

BN_EPS = 1e-5
BN_MOMENTUM = 0.1
S2D_PAD = 2   # zero pixels kept on either side of every row of the space-to-depth input planes (= the 4x4 stem's padding)

# name -> (fwd_npass, fwd_bf16, bwd_npass): forward planes fp16 (hi/lo) or bf16; the backbone's gradient planes take the
# forward planes' format (fp16: hi/lo of dY * 2^k, see Plan), the head's gradient planes are bf16
PRECISIONS = {
    "parity": (3, 0, 3),   # fp16 hi/lo split forward (fp32-grade), hi/lo split backward
    "mixed": (3, 0, 1),    # fp32-grade forward (same logits/loss/queue as parity), single-pass backward
    "fast": (1, 1, 1),     # single-pass bf16 everywhere (does NOT meet the 1e-3 parity bar)
}


def _round8(c):
    return (c + 7) // 8 * 8


class Launch(namedtuple("Launch", "fn args")):
    """One launch of a plan, fn(*args, stream), which unpacks as (fn, args).  It runs on stream lane `lane` (0: the
    caller's current stream, 1..3: the engine's own streams) once that lane has waited for `wait`, and it is `kernels`
    kernels of the library (L.kernels_of, set by the plan once the launch's workspace is known)."""

    def __new__(cls, fn, args, lane=0, wait=None):
        r = super().__new__(cls, fn, args)
        r.lane, r.wait, r.kernels = lane, wait, None
        return r


# Launch.wait.  The Inception branches of a Mixed block run on lanes 1..3 from the block's fork point, an event that
# lane 0 records before the block's first launch.
FORK = "fork"          # lane 0 records the fork point, the launch's lane waits for it
AT_FORK = "at fork"    # the fork point (not lane 0's current point: work queued there since must not delay the branch)
AFTER1 = "after 1"     # the fork point, then the work lane 1 has been given so far
AFTER0 = "after 0"     # the work lane 0 has been given so far
JOIN = "join"          # on lane 0: every lane that waited for something since the last JOIN


# ---------------------------------------------------------------------------------------------
# symbolic graph
# ---------------------------------------------------------------------------------------------
class TensorSpec:
    def __init__(self, name, C, dims_fn, pending):
        self.name, self.C, self.dims_fn, self.pending = name, C, dims_fn, pending
        self.bn_members = []   # (bn module name, coff, C) in channel order
        self.relu = 1 if pending else 0
        self.residual = None   # TensorSpec added before the ReLU (ResNet bottleneck output)
        self.gates = []        # S3D-G: (SelfGating module name, coff, C) per branch slice of a SepInception output
        self.lane, self.wait = 0, None   # as a BatchNorm item: lane of its launches, wait of the first (Launch)


class ConvSpec:
    def __init__(self, name, src, dst, dst_coff, cin, cout, k, s, p, bias=None, need_dgrad=True):
        self.name, self.src, self.dst, self.dst_coff = name, src, dst, dst_coff
        self.cin, self.cout, self.k, self.s, self.p = cin, cout, k, s, p
        self.bias, self.need_dgrad = bias, need_dgrad
        # what the kernels see; differs from the parameter's own shape only for the space-to-depth stem
        self.s2d = False
        self.cin_eff, self.k_eff, self.s_eff, self.p_eff = cin, k, s, p
        # channel slice of the source tensor this conv reads (default: all of it)
        self.src_coff, self.src_C = 0, src.C
        # parameter names whose (adjacent) [cout_i, cin, 1, 1, 1] weights this conv uses as one [sum cout_i, cin] matrix
        self.weight_names = [name]
        self.lane, self.wait = 0, None


class PoolSpec:
    def __init__(self, name, src, dst, k, s, p):
        self.name, self.src, self.dst, self.k, self.s, self.p = name, src, dst, k, s, p
        self.fused = False   # pools straight from its source's conv output (see Graph._fuse_pools)
        self.lane, self.wait = 0, None


# (kernel, stride) of the pools coclr_maxpool_fwd can run from a conv output (coclr_pool_t.y)
FUSED_POOL_WINDOWS = {((1, 3, 3), (1, 2, 2)), ((3, 3, 3), (2, 2, 2)), ((2, 2, 2), (2, 2, 2))}


def _conv_out(d, k, s, p):
    return (d + 2 * p - k) // s + 1


class Graph:
    """Shape-independent description of the encoder: tensors, convs, pools in forward order."""

    def __init__(self, stages, first_channel=3, head_dim=None, feature_size=S3D_FEATURE_SIZE, bb_prefix="",
                 stem_s2d=True, pooled=False):
        """pooled (only without a head): the pass ends with the average-pooled feature [B, feature_size] and its
        backward starts from that feature's gradient (LinearClassifier's backbone)."""
        assert not (pooled and head_dim is not None)
        self.pooled = pooled
        self.tensors, self.items = [], []   # items: ("conv", ConvSpec) | ("pool", PoolSpec) | ("bn", TensorSpec)
        self.first_channel = first_channel
        self.head_dim, self.feature_size = head_dim, feature_size
        pre = bb_prefix
        st0 = stages[0]
        # stride-2 7x7 RGB stem as a stride-1 4x4 conv over a space-to-depth input (16 channels / pixel): 16 taps of
        # 32-byte granules instead of 49 taps of 16-byte granules
        if st0[0] == "st":
            s2d_ok = st0[4] == 7 and st0[5] == 2 and st0[7] == 3
        elif st0[0] == "convbn":
            s2d_ok = tuple(st0[5][1:]) == (7, 7) and tuple(st0[6][1:]) == (2, 2) and tuple(st0[7][1:]) == (3, 3)
        else:
            s2d_ok = False
        self.stem_s2d = bool(stem_s2d and s2d_ok and 4 * first_channel <= 16)
        if self.stem_s2d:
            x = self._tensor("input", 16, lambda d: (d[0], d[1] // 2, d[2] // 2), pending=False)
        else:
            x = self._tensor("input", _round8(first_channel), lambda d: d, pending=False)
        self.input = x
        first_conv = True
        for stg in stages:
            kind = stg[0]
            if kind == "st":
                _, name, cin, cout, k, ss, ts, pad = stg
                x = self._st(pre + name, x, None, 0, cin, cout, k, ss, ts, pad, need_dgrad=not first_conv)
                first_conv = False
            elif kind == "basic":
                _, name, cin, cout = stg
                y = self._tensor(pre + name, cout, self._same(x))
                self._conv(pre + name + ".conv", x, y, 0, cin, cout, (1, 1, 1), (1, 1, 1), (0, 0, 0))
                y.bn_members.append((pre + name + ".bn", 0, cout))
                self.items.append(("bn", y))
                x = y
            elif kind == "pool":
                _, name, k, s, p = stg
                x = self._pool(pre + name, x, k, s, p)
            elif kind == "convbn":
                _, cname, bname, cin, cout, k, s, p = stg
                s2d = first_conv and self.stem_s2d and x is self.input
                if s2d:
                    f = x.dims_fn
                    dims = (lambda d, f=f, k=k, s=s, p=p: (_conv_out(f(d)[0], k[0], s[0], p[0]), f(d)[1], f(d)[2]))
                else:
                    dims = self._after(x, k, s, p)
                y = self._tensor(pre + cname + ".out", cout, dims)
                cv = self._conv(pre + cname, x, y, 0, cin, cout, tuple(k), tuple(s), tuple(p), need_dgrad=not first_conv)
                if s2d:
                    cv.s2d, cv.cin_eff = True, 4 * cin
                    cv.k_eff, cv.s_eff, cv.p_eff = (k[0], 4, 4), (s[0], 1, 1), (p[0], 2, 2 - S2D_PAD)
                first_conv = False
                y.bn_members.append((pre + bname, 0, cout))
                self.items.append(("bn", y))
                x = y
            elif kind == "bottleneck":
                _, name, inplanes, planes, stride, is3d, has_ds = stg
                x = self._bottleneck(pre + name, x, inplanes, planes, stride, is3d, has_ds)
            elif kind == "mixed":
                name, cin, planes = stg[1:4]
                x = self._mixed(pre + name, x, cin, planes, gating=len(stg) > 4 and bool(stg[4]))
            else:
                raise ValueError(kind)
        self.backbone_out = x
        self._fuse_pools()

    def _fuse_pools(self):
        """A max-pool whose input is a plain BatchNorm(+ReLU) output -- no gating, no residual -- that nothing else
        reads pools straight from the conv output: its BatchNorm item only finalizes the statistics and the pool applies
        BatchNorm + ReLU while it loads, so the input's planes are never written or read.  The Inception branch-3
        pools stay on the planes: their input also feeds convolutions."""
        readers = {}
        for kind, it in self.items:
            if kind in ("conv", "pool"):
                readers[it.src.index] = readers.get(it.src.index, 0) + 1
        for t in self.tensors:
            if t.residual is not None:
                readers[t.residual.index] = readers.get(t.residual.index, 0) + 1
        for kind, it in self.items:
            if kind == "pool":
                src = it.src
                it.fused = (src.pending and not src.gates and src.residual is None and readers[src.index] == 1
                            and src is not self.backbone_out and (tuple(it.k), tuple(it.s)) in FUSED_POOL_WINDOWS)

    # -- helpers --
    def _tensor(self, name, C, dims_fn, pending=True):
        t = TensorSpec(name, C, dims_fn, pending)
        t.index = len(self.tensors)
        self.tensors.append(t)
        return t

    @staticmethod
    def _same(src):
        return src.dims_fn

    @staticmethod
    def _after(src, k, s, p):
        f = src.dims_fn
        return lambda d: tuple(_conv_out(v, kk, ss, pp) for v, kk, ss, pp in zip(f(d), k, s, p))

    def _conv(self, name, src, dst, dst_coff, cin, cout, k, s, p, need_dgrad=True):
        c = ConvSpec(name, src, dst, dst_coff, cin, cout, k, s, p, need_dgrad=need_dgrad)
        self.items.append(("conv", c))
        return c

    def _st(self, name, x, dst, dst_coff, cin, cout, k, ss, ts, pad, need_dgrad=True, src_coff=0):
        k1, s1, p1 = (1, k, k), (1, ss, ss), (0, pad, pad)
        k2, s2, p2 = (k, 1, 1), (ts, 1, 1), (pad, 0, 0)
        s2d = (not need_dgrad) and self.stem_s2d and x is self.input
        mid = self._tensor(name + ".mid", cout, self._same(x) if s2d else self._after(x, k1, s1, p1))
        cv = self._conv(name + ".conv1", x, mid, 0, cin, cout, k1, s1, p1, need_dgrad=need_dgrad)
        if src_coff or cin != x.C and x is not self.input:
            cv.src_coff, cv.src_C = src_coff, cin
        if s2d:
            cv.s2d, cv.cin_eff, cv.k_eff, cv.s_eff, cv.p_eff = True, 4 * cin, (1, 4, 4), (1, 1, 1), (0, 2, 2 - S2D_PAD)
        mid.bn_members.append((name + ".bn1", 0, cout))
        self.items.append(("bn", mid))
        own = dst is None
        if own:
            dst = self._tensor(name, cout, self._after(mid, k2, s2, p2))
        self._conv(name + ".conv2", mid, dst, dst_coff, cout, cout, k2, s2, p2)
        dst.bn_members.append((name + ".bn2", dst_coff, cout))
        if own:
            self.items.append(("bn", dst))
        return dst

    def _pool(self, name, x, k, s, p):
        y = self._tensor(name, x.C, self._after(x, k, s, p), pending=False)
        self.items.append(("pool", PoolSpec(name, x, y, k, s, p)))
        return y

    def _mixed(self, name, x, cin, planes, gating=False):
        o0, o1a, o1b, o2a, o2b, o3b = planes
        cat = self._tensor(name, o0 + o1b + o2b + o3b, self._same(x))
        if gating:   # SepInception(gating=True): one SelfGating per branch output (backbone/s3dg.py:107-112,125-129)
            cat.gates = [(name + ".gating_b0", 0, o0), (name + ".gating_b1", o0, o1b),
                         (name + ".gating_b2", o0 + o1b, o2b), (name + ".gating_b3", o0 + o1b + o2b, o3b)]
        one = ((1, 1, 1), (1, 1, 1), (0, 0, 0))
        # the 1x1x1 convs that open branches 1 and 2 read the same input: they run as ONE conv (N = o1a + o2a instead
        # of e.g. 96 and 16 output channels) into one buffer that the two branches slice
        t12 = self._tensor(name + ".b12a", o1a + o2a, self._same(x))
        n = len(self.items)   # lane 1: fused 1x1 conv + its BN, then branch 1
        cv = self._conv(name + ".branch1.0.conv", x, t12, 0, cin, o1a + o2a, *one)
        cv.weight_names, cv.couts = [name + ".branch1.0.conv", name + ".branch2.0.conv"], [o1a, o2a]
        t12.bn_members += [(name + ".branch1.0.bn", 0, o1a), (name + ".branch2.0.bn", o1a, o2a)]
        self.items.append(("bn", t12))
        self._on_lane(n, 1, FORK)
        n = len(self.items)   # lane 2: branch 2 starts once the shared buffer is ready
        self._st(name + ".branch2.1", t12, cat, o0 + o1b, o2a, o2b, 3, 1, 1, 1, src_coff=o1a)
        self._on_lane(n, 2, AFTER1)
        n = len(self.items)
        self._st(name + ".branch1.1", t12, cat, o0, o1a, o1b, 3, 1, 1, 1, src_coff=0)
        self._on_lane(n, 1, None)
        self._conv(name + ".branch0.0.conv", x, cat, 0, cin, o0, *one)
        cat.bn_members.append((name + ".branch0.0.bn", 0, o0))
        n = len(self.items)
        tp = self._pool(name + ".branch3.0", x, (3, 3, 3), (1, 1, 1), (1, 1, 1))
        self._conv(name + ".branch3.1.conv", tp, cat, o0 + o1b + o2b, cin, o3b, *one)
        cat.bn_members.append((name + ".branch3.1.bn", o0 + o1b + o2b, o3b))
        self._on_lane(n, 3, AT_FORK)
        # the branches were issued out of channel order; the per-tensor BatchNorm needs its members' parameters laid
        # out in channel order (one gamma / beta vector for the whole concat buffer)
        cat.bn_members.sort(key=lambda m: m[1])
        cat.wait = JOIN
        self.items.append(("bn", cat))
        return cat

    def _on_lane(self, start, lane, wait):
        """Put the items appended since items[start] on stream lane `lane`, the first of them waiting for `wait`."""
        for _, spec in self.items[start:]:
            spec.lane = lane
        self.items[start][1].wait = wait

    def _bottleneck(self, name, x, inplanes, planes, stride, is3d, has_ds):
        """Bottleneck2d / Bottleneck3d (backbone/resnet_2d3d.py:46-131): conv1 (1x1x1 or (3,1,1)) -> conv2 (1,3,3) with
        the spatial stride -> conv3 1x1x1 (x4); out = relu(bn3(.) + residual), residual = x or bn(downsample conv(x))."""
        one = ((1, 1, 1), (1, 1, 1), (0, 0, 0))
        k1, s1, p1 = ((3, 1, 1), (1, 1, 1), (1, 0, 0)) if is3d else one
        t1 = self._tensor(name + ".t1", planes, self._after(x, k1, s1, p1))
        self._conv(name + ".conv1", x, t1, 0, inplanes, planes, k1, s1, p1)
        t1.bn_members.append((name + ".bn1", 0, planes))
        self.items.append(("bn", t1))
        k2, s2, p2 = (1, 3, 3), (1, stride, stride), (0, 1, 1)
        t2 = self._tensor(name + ".t2", planes, self._after(t1, k2, s2, p2))
        self._conv(name + ".conv2", t1, t2, 0, planes, planes, k2, s2, p2)
        t2.bn_members.append((name + ".bn2", 0, planes))
        self.items.append(("bn", t2))
        out = self._tensor(name, 4 * planes, self._same(t2))
        self._conv(name + ".conv3", t2, out, 0, planes, 4 * planes, *one)
        out.bn_members.append((name + ".bn3", 0, 4 * planes))
        if has_ds:
            ds = self._tensor(name + ".ds", 4 * planes, self._same(t2))
            ds.relu = 0
            self._conv(name + ".downsample.0", x, ds, 0, inplanes, 4 * planes, (1, 1, 1), (1, stride, stride), (0, 0, 0))
            ds.bn_members.append((name + ".downsample.1", 0, 4 * planes))
            self.items.append(("bn", ds))
            out.residual = ds
        else:
            out.residual = x
        self.items.append(("bn", out))
        return out

    # -- parameter inventory (names relative to the encoder: backbone under bb_prefix, head '2.', '4.') --
    def param_layout(self):
        """[(name, shape)] in flat-buffer order; BN members of one tensor are contiguous (all gammas, then
        all betas) so that BatchNorm kernels address a whole concat buffer at once."""
        out = []
        for kind, it in self.items:
            if kind == "conv":
                if len(it.weight_names) == 1:
                    out.append((it.name + ".weight", (it.cout, it.cin) + tuple(it.k)))
                else:   # fused convs: the member weights follow each other in the flat buffer (see ParamStore.view_span)
                    for wn, co in zip(it.weight_names, it.couts):
                        out.append((wn + ".weight", (co, it.cin) + tuple(it.k)))
        for kind, it in self.items:
            if kind == "bn":
                for nm, _, c in it.bn_members:
                    out.append((nm + ".weight", (c,)))
                for nm, _, c in it.bn_members:
                    out.append((nm + ".bias", (c,)))
        for kind, it in self.items:
            if kind == "bn":
                for nm, _, c in it.gates:      # nn.Linear(c, c) of a SelfGating
                    out += [(nm + ".fc.weight", (c, c)), (nm + ".fc.bias", (c,))]
        if self.head_dim is not None:
            fs = self.feature_size
            out += [("2.weight", (fs, fs, 1, 1, 1)), ("2.bias", (fs,)),
                    ("4.weight", (self.head_dim, fs, 1, 1, 1)), ("4.bias", (self.head_dim,))]
        return out

    def buffer_layout(self):
        """[(name, C)] for running_mean (same order for running_var), tensor-contiguous."""
        out = []
        for kind, it in self.items:
            if kind == "bn":
                for nm, _, c in it.bn_members:
                    out.append((nm, c))
        return out


# ---------------------------------------------------------------------------------------------
# flat parameter storage
# ---------------------------------------------------------------------------------------------
class ParamStore:
    """One flat fp32 buffer for a module's parameters (+ flat grad, flat BN running stats)."""

    def __init__(self, layout, device, buffer_layout=()):
        """layout: [(name, shape)] of the parameters in flat-buffer order, each starting 16-byte aligned;
        buffer_layout: [(name, C)] of the BatchNorms whose running statistics and num_batches_tracked live in flat
        buffers too.  A Graph as `layout` stands for its param_layout() and buffer_layout()."""
        if isinstance(layout, Graph):
            layout, buffer_layout = layout.param_layout(), layout.buffer_layout()
        self.device = device
        self.offsets = {}
        off = 0
        for name, shape in layout:
            n = 1
            for s in shape:
                n *= s
            self.offsets[name] = (off, n, shape)
            off += (n + 3) // 4 * 4
        self.numel = off
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.grad = torch.zeros(off, dtype=torch.float32, device=device)
        self.buf_offsets = {}
        boff = 0
        for name, c in buffer_layout:
            self.buf_offsets[name] = (boff, c)
            boff += c
        self.running_mean = torch.zeros(boff, dtype=torch.float32, device=device)
        self.running_var = torch.ones(boff, dtype=torch.float32, device=device)
        self.nbt = torch.zeros(len(self.buf_offsets), dtype=torch.long, device=device)
        self.params = []   # the bound nn.Parameters in layout order (bind_module)

    def owns(self, t):
        """Whether tensor t lies in the flat parameter buffer (its module's parameters are still views of it)."""
        off = t.data_ptr() - self.flat.data_ptr()
        return t.device == self.flat.device and 0 <= off < 4 * self.numel

    def view(self, name, grad=False):
        off, n, shape = self.offsets[name]
        return (self.grad if grad else self.flat)[off:off + n].view(shape)

    def view_span(self, names, grad=False):
        """One [sum cout_i, cin, kt, kh, kw] view over parameters that follow each other without gaps in the flat buffer."""
        off0, _, shape0 = self.offsets[names[0]]
        end, rows = off0, 0
        for nm in names:
            off, n, shape = self.offsets[nm]
            if off != end or tuple(shape[1:]) != tuple(shape0[1:]):
                raise RuntimeError("parameters %s are not adjacent in the flat buffer" % (names,))
            end, rows = off + n, rows + shape[0]
        return (self.grad if grad else self.flat)[off0:end].view((rows,) + tuple(shape0[1:]))

    def bind_module(self, named_params, named_buffers):
        """Copy the module's current values in and rebind every Parameter / BN buffer to a view."""
        with torch.no_grad():
            self.params = []
            for name in self.offsets:
                p = named_params[name]
                v = self.view(name)
                v.copy_(p.detach().to(self.device))
                p.data = v
                p.grad = None
                self.params.append((name, p))
            nbt_host = []
            for name, (boff, c) in self.buf_offsets.items():
                for suffix, flat in ((".running_mean", self.running_mean), (".running_var", self.running_var)):
                    b = named_buffers[name + suffix]
                    assert b.device == flat.device, "move the module to the CUDA device before the first forward"
                    v = flat[boff:boff + c]
                    v.copy_(b)
                    b.set_(v.untyped_storage(), v.storage_offset(), v.shape, v.stride())
                nbt_host.append(named_buffers[name + ".num_batches_tracked"])
            if nbt_host:
                self.nbt.copy_(torch.stack([t.detach().reshape(()) for t in nbt_host]).to(self.nbt.device))
            for i, nb in enumerate(nbt_host):
                nb.set_(self.nbt.untyped_storage(), i, (), ())

    def attach_grads(self):
        """Make the .grad of every bound parameter that requires one its view of the flat gradient.  When the first
        such parameter's .grad is not that view (None after zero_grad(set_to_none=True), or replaced), the gradients
        count as cleared: the flat gradient is zeroed first.  Every way of clearing gradients clears all of them."""
        trained = [(name, p) for name, p in self.params if p.requires_grad]
        if not trained:
            return
        name, p = trained[0]
        if p.grad is None or p.grad.data_ptr() != self.view(name, grad=True).data_ptr():
            self.grad.zero_()
            for name, p in trained:
                p.grad = self.view(name, grad=True)


def bind_engine(engine, probe, module, make_graph, precision):
    """The engine that runs `module`'s parameters: `engine` itself while its store still owns `probe` (one of the
    module's parameter tensors), else a new engine over a new store of make_graph()'s layout, with the module's
    parameters and BatchNorm buffers re-bound to views of the store's flat buffers (first call, .cuda(), .to())."""
    if not probe.is_cuda:
        raise L.CoclrError("coclr_b200 runs on CUDA (sm_90a) only; move the module to the GPU")
    if engine is not None and engine.store.owns(probe):
        return engine
    graph = make_graph()
    store = ParamStore(graph, probe.device)
    store.bind_module(dict(module.named_parameters()), dict(module.named_buffers()))
    return EncoderEngine(store, graph, precision)


# ---------------------------------------------------------------------------------------------
# shape-specific plan
# ---------------------------------------------------------------------------------------------
class _Act:
    __slots__ = ("spec", "dims", "data", "pl", "grad", "dy", "scale", "shift", "mean", "rstd", "ssum", "ssq", "idx",
                 "bsums", "grad_written", "M", "dy_scale", "bamax", "gmean", "gate", "dgate", "dmean")


class _PoolInputView:
    """Stands in for the planes of a tensor whose max-pool reads the conv output itself, which are never stored:
    value() recomputes relu(bn(y)) from the conv output and the published scale / shift, bit-identical to what the
    pool compared (for inspection; nothing on the training path reads it)."""

    def __init__(self, a):
        self.a = a

    def value(self):
        a = self.a
        pl = ops.Planes(a.data.shape, 0, a.data.device)
        ops.split_into(a.data, pl, scale=a.scale, shift=a.shift, relu=a.spec.relu)
        return pl.value()


def _count_kernels(records):
    """Set each record's kernel count (L.kernels_of); returns their total."""
    for r in records:
        r.kernels = L.kernels_of(r.fn, r.args)
    return sum(r.kernels for r in records)


class Plan:
    """Buffers + launch lists for one (B, T, H, W, training) configuration."""

    def __init__(self, eng, B, T, H, W, training, with_backward):
        self.eng, self.B, self.dims0, self.training, self.with_backward = eng, B, (T, H, W), training, with_backward
        g, dev = eng.graph, eng.store.device
        lib = L.load()
        self.keep = []          # keeps ctypes structs / tensors alive
        self.fwd, self.bwd = [], []   # Launch records
        self.graphs = {}      # captured CUDA graphs of the launch lists
        nsm = L.num_sms(dev)
        fnp, fbf, bnp = PRECISIONS[eng.precision]
        # gradient planes: with fp16 forward planes dY is stored as fp16 hi/lo of dY * 2^k (k per tensor and step, chosen
        # by coclr_bn_bwd from the data's range) so that the weight-gradient GEMM pairs it with the forward planes --
        # wgmma wants one 16-bit format for both operands -- instead of a bf16 twin of every activation
        gbf = 1 if fbf else 0
        # source tensor index -> its max-pool that reads the conv output (fp16 planes only: that pool splits into fp16)
        fused_pool = {it.src.index: it for kind, it in g.items if kind == "pool" and it.fused and not fbf}
        self.fused_pools = [it.name for it in fused_pool.values()]
        # ---- activations ----
        acts = {}
        n_stat = sum(t.C for t in g.tensors if t.pending)
        self.stats = torch.zeros(2 * n_stat, dtype=torch.float64, device=dev)
        self.aff = torch.zeros(4 * n_stat, dtype=torch.float32, device=dev)  # scale, shift, mean, rstd
        so = 0
        for t in g.tensors:
            a = _Act()
            a.spec, a.dims = t, t.dims_fn((T, H, W))
            a.M = B * a.dims[0] * a.dims[1] * a.dims[2]
            shape = (B,) + a.dims + (t.C,)
            # the space-to-depth input keeps the stem's horizontal zero padding in memory (rows of W + 2*S2D_PAD pixels,
            # written once here and never touched by the packing kernel): see coclr_pack_input_s2d
            padded = g.stem_s2d and t is g.input
            if padded:
                shape = (B,) + a.dims[:2] + (a.dims[2] + 2 * S2D_PAD, t.C)
            # what every forward consumer reads, and the weight-gradient GEMM (same 16-bit format as dY)
            if t.index in fused_pool:
                a.pl = _PoolInputView(a)
            else:
                a.pl = ops.Planes(shape, fbf, dev, lo=fnp > 1, zero=padded)
            a.data = a.grad = a.dy = a.idx = a.bsums = a.dy_scale = a.bamax = None
            a.gmean = a.gate = a.dgate = a.dmean = None
            a.grad_written = False
            if t.pending:
                a.data = torch.empty(shape, dtype=torch.float32, device=dev)   # raw conv output (pre-BN)
                a.ssum = self.stats[so:so + t.C]
                a.ssq = self.stats[n_stat + so:n_stat + so + t.C]
                a.scale = self.aff[so:so + t.C]
                a.shift = self.aff[n_stat + so:n_stat + so + t.C]
                a.mean = self.aff[2 * n_stat + so:2 * n_stat + so + t.C]
                a.rstd = self.aff[3 * n_stat + so:3 * n_stat + so + t.C]
                so += t.C
            else:
                a.ssum = a.ssq = a.scale = a.shift = a.mean = a.rstd = None
            if with_backward and t is not g.input:
                a.grad = torch.empty(shape, dtype=torch.float32, device=dev)
                if t.pending:
                    a.dy = ops.Planes(shape, gbf, dev, lo=bnp > 1)
                    a.dy_scale = torch.ones(2, dtype=torch.float32, device=dev)      # (s, 1/s) written by coclr_bn_bwd
            acts[t.index] = a
        self.acts = acts
        self.input = acts[g.input.index]
        st = eng.store

        def src_w(a):
            return a.dims[2] + (2 * S2D_PAD if (g.stem_s2d and a.spec is g.input) else 0)

        def src_of(a, it=None):
            coff, cc = (it.src_coff, it.src_C) if it is not None else (0, a.spec.C)
            return a.pl.src(coff, cc, a.dims[0], a.dims[1], src_w(a))

        # which channel ranges of a tensor's gradient buffer already hold a value (first writer stores, later ones add)
        grad_ranges = {}

        def grad_seen(a, coff=0, cc=None):
            key = (coff, a.spec.C if cc is None else cc)
            seen = key in grad_ranges.setdefault(a.spec.index, set()) or (0, a.spec.C) in grad_ranges[a.spec.index]
            grad_ranges[a.spec.index].add(key)
            a.grad_written = True
            return seen

        def twin_ptrs(pl, plw):
            if plw is None or plw is pl:
                return None, None
            return L.dptr(plw.hi), L.dptr(plw.lo)

        def split_op(x, planes, M, Cc, scale, shift, relu, twin=None, bn=None, res=None, lane=0):
            t_hi, t_lo = twin_ptrs(planes, twin)
            sp = L.Split(L.dptr(x), x.shape[-1], 0, Cc, M, L.dptr(scale), L.dptr(shift), int(bool(relu)),
                         L.dptr(planes.hi), L.dptr(planes.lo), planes.ld, 0, planes.bf16, t_hi, t_lo,
                         bn if bn is not None else L.BnFinalize(),
                         L.dptr(res.hi) if res is not None else None, L.dptr(res.lo) if res is not None else None,
                         res.ld if res is not None else 0, 0)
            self.keep.append(sp)
            return Launch(lib.coclr_affine_split, (C.byref(sp), nsm), lane)

        # ---- forward ----
        for kind, it in g.items:
            n_before = len(self.fwd)
            if kind == "conv":
                sa, da = acts[it.src.index], acts[it.dst.index]
                geom = ops.Geometry(it.k_eff, it.s_eff, it.p_eff)
                pw = eng.packed_fwd[it.name]
                cv = ops.make_conv(src_of(sa, it), fbf, geom.c(0), B, da.dims, pw, da.data, it.dst_coff,
                                   stats_sum=da.ssum[it.dst_coff:] if training else None,
                                   stats_sq=da.ssq[it.dst_coff:] if training else None, npass=fnp)
                self.keep.append(cv)
                self.fwd.append(Launch(lib.coclr_conv_igemm, (C.byref(cv), nsm), it.lane))
            elif kind == "pool":
                sa, da = acts[it.src.index], acts[it.dst.index]
                geom = ops.Geometry(it.k, it.s, it.p)
                if with_backward:
                    da.idx = torch.empty(da.M * it.dst.C, dtype=torch.uint8, device=dev)
                fused = it.src.index in fused_pool
                pl = L.Pool(None if fused else L.dptr(sa.pl.hi), None if fused else L.dptr(sa.pl.lo), it.src.C, 0,
                            L.dptr(da.pl.hi), L.dptr(da.pl.lo), it.dst.C, 0, None, None, L.dptr(da.idx), B, it.dst.C,
                            sa.dims[0], sa.dims[1], sa.dims[2], da.dims[0], da.dims[1], da.dims[2], geom.c(0),
                            None, None, 0)
                if fused:   # BatchNorm + ReLU applied while loading the conv output
                    pl.y, pl.scale, pl.shift, pl.relu = L.dptr(sa.data), L.dptr(sa.scale), L.dptr(sa.shift), it.src.relu
                self.keep.append(pl)
                self.fwd.append(Launch(lib.coclr_maxpool_fwd, (C.byref(pl),), it.lane))
            elif kind == "bn":
                a = acts[it.index]
                first = it.bn_members[0][0]
                goff = st.offsets[first + ".weight"][0]
                boff_b = st.offsets[first + ".bias"][0]
                rboff = st.buf_offsets[first][0]
                bf = L.BnFinalize(L.dptr(a.ssum), L.dptr(a.ssq), a.M,
                                  L.dptr(st.flat[goff:]), L.dptr(st.flat[boff_b:]),
                                  L.dptr(st.running_mean[rboff:]), L.dptr(st.running_var[rboff:]),
                                  BN_MOMENTUM, BN_EPS, int(training), L.dptr(a.scale), L.dptr(a.shift),
                                  L.dptr(a.mean), L.dptr(a.rstd), it.C)
                if it.index in fused_pool:
                    # the finalize alone: the max-pool that is this tensor's only consumer applies it (no planes)
                    sp = L.Split(L.dptr(a.data), it.C, 0, it.C, a.M, None, None, it.relu, None, None, it.C, 0, 0,
                                 None, None, bf)
                    self.keep.append(sp)
                    self.fwd.append(Launch(lib.coclr_affine_split, (C.byref(sp), nsm), it.lane))
                else:
                    # BatchNorm finalize is fused into the apply+split launch
                    res = acts[it.residual.index].pl if it.residual is not None else None
                    self.fwd.append(split_op(a.data, a.pl, a.M, it.C, None, None, it.relu, bn=bf, res=res, lane=it.lane))
                if it.gates:
                    # S3D-G feature gating of the block output: the planes written above are scaled in place by
                    # sigmoid(fc(mean_thw)) per clip and channel (csrc/gating.cu)
                    Pn = a.dims[0] * a.dims[1] * a.dims[2]
                    a.gmean = torch.empty(B, it.C, dtype=torch.float32, device=dev)
                    a.gate = torch.empty(B, it.C, dtype=torch.float32, device=dev)
                    self.fwd.append(Launch(lib.coclr_gate_mean, (L.dptr(a.pl.hi), L.dptr(a.pl.lo), a.pl.bf16, a.pl.ld, B,
                                                              Pn, it.C, L.dptr(a.gmean)), it.lane))
                    for nm, coff, c in it.gates:
                        self.fwd.append(Launch(lib.coclr_gate_fc, (L.dptr(a.gmean), L.dptr(st.view(nm + ".fc.weight")),
                                                                L.dptr(st.view(nm + ".fc.bias")), L.dptr(a.gate), B, it.C,
                                                                coff, c), it.lane))
                    self.fwd.append(Launch(lib.coclr_gate_apply, (L.dptr(a.pl.hi), L.dptr(a.pl.lo), a.pl.bf16, a.pl.ld, B,
                                                               Pn, it.C, L.dptr(a.gate)), it.lane))
            self.fwd[n_before].wait = it.wait   # the item's first launch waits
        # ---- head ----
        out = acts[g.backbone_out.index]
        self.backbone_out = out
        if g.head_dim is not None:
            fs, hd = g.feature_size, g.head_dim
            Pn = out.dims[0] * out.dims[1] * out.dims[2]
            f32 = dict(dtype=torch.float32, device=dev)
            self.feat = torch.empty(B, 1, 1, 1, fs, **f32)
            self.h1 = torch.empty(B, 1, 1, 1, fs, **f32)
            self.h2 = torch.empty(B, 1, 1, 1, hd, **f32)
            self.q = torch.empty(B, hd, **f32)
            self.inv_norm = torch.empty(B, **f32)
            self.ones = torch.ones(fs, **f32)
            self.feat_pl = ops.Planes((B, 1, 1, 1, fs), fbf, dev, lo=fnp > 1)
            self.h1_pl = ops.Planes((B, 1, 1, 1, fs), fbf, dev, lo=fnp > 1)
            mk_twin = with_backward and not fbf
            self.feat_plw = ops.Planes((B, 1, 1, 1, fs), 1, dev, lo=bnp > 1) if mk_twin else self.feat_pl
            self.h1_plw = ops.Planes((B, 1, 1, 1, fs), 1, dev, lo=bnp > 1) if mk_twin else self.h1_pl
            self.fwd.append(Launch(lib.coclr_avgpool_fwd, (L.dptr(out.pl.hi), L.dptr(out.pl.lo), out.pl.bf16, out.spec.C,
                                                        0, L.dptr(self.feat), B, Pn, fs)))
            self.fwd.append(split_op(self.feat, self.feat_pl, B, fs, None, None, False, self.feat_plw))
            one = ops.Geometry((1, 1, 1))
            b2, b4 = st.view("2.bias"), st.view("4.bias")
            s_feat = self.feat_pl.src(0, fs, 1, 1, 1)
            s_h1 = self.h1_pl.src(0, fs, 1, 1, 1)
            c1 = ops.make_conv(s_feat, fbf, one.c(0), B, (1, 1, 1), eng.packed_fwd["2"], self.h1, npass=fnp)
            c2 = ops.make_conv(s_h1, fbf, one.c(0), B, (1, 1, 1), eng.packed_fwd["4"], self.h2, npass=fnp)
            self.keep += [c1, c2, s_feat, s_h1]
            self.fwd.append(Launch(lib.coclr_conv_igemm, (C.byref(c1), nsm)))
            self.fwd.append(split_op(self.h1, self.h1_pl, B, fs, self.ones, b2, True, self.h1_plw))   # bias + ReLU
            self.fwd.append(Launch(lib.coclr_conv_igemm, (C.byref(c2), nsm)))
            self.fwd.append(Launch(lib.coclr_l2norm_fwd, (L.dptr(self.h2), L.dptr(b4), L.dptr(self.q), L.dptr(self.inv_norm),
                                                       B, hd)))
        elif g.pooled:
            fs, Pn = g.feature_size, out.dims[0] * out.dims[1] * out.dims[2]
            self.feat = torch.empty(B, fs, dtype=torch.float32, device=dev)
            self.fwd.append(Launch(lib.coclr_avgpool_fwd, (L.dptr(out.pl.hi), L.dptr(out.pl.lo), out.pl.bf16, out.spec.C,
                                                        0, L.dptr(self.feat), B, Pn, fs)))
        self.fwd_kernels, self.bwd_kernels = _count_kernels(self.fwd), 0
        if not with_backward:
            return
        # ---- backward ----
        bw = self.bwd
        # The weight gradients that share the workspace wg_ws (sized at the end) run one after another on lane 1, each
        # once lane 0 has produced its dY: nothing later in the pass reads dW, and small layers leave most SMs idle, so
        # the two chains overlap.
        self.wgrads, self.s2d_wgrads = [], []   # coclr_wgrad_t structs of the shared and the own-workspace launches
        if g.head_dim is not None:
            self.dq = torch.empty(B, hd, **f32)
            self.dh2 = torch.empty(B, 1, 1, 1, hd, **f32)
            self.dh1 = torch.empty(B, 1, 1, 1, fs, **f32)
            self.dfeat = torch.empty(B, 1, 1, 1, fs, **f32)
            self.dh2_pl = ops.Planes((B, 1, 1, 1, hd), 1, dev, lo=bnp > 1)
            self.dh1_pl = ops.Planes((B, 1, 1, 1, fs), 1, dev, lo=bnp > 1)
            bw.append(Launch(lib.coclr_l2norm_bwd, (L.dptr(self.q), L.dptr(self.dq), L.dptr(self.inv_norm), L.dptr(self.dh2),
                                                 L.dptr(st.view("4.bias", grad=True)), B, hd)))
            bw.append(split_op(self.dh2, self.dh2_pl, B, hd, None, None, False))
            s_dh2 = self.dh2_pl.src(0, hd, 1, 1, 1)
            s_dh1 = self.dh1_pl.src(0, fs, 1, 1, 1)
            sw_h1 = self.h1_plw.src(0, fs, 1, 1, 1)
            sw_feat = self.feat_plw.src(0, fs, 1, 1, 1)
            wg2 = L.Wgrad(sw_h1, one.c(0), s_dh2, B, 1, 1, 1, hd, fs, L.dptr(st.view("4.weight", grad=True)), bnp, 1, 1, 1)
            dg2 = ops.make_conv(s_dh2, 1, one.c(1), B, (1, 1, 1), eng.packed_bwd["4"], self.dh1, npass=bnp)
            wg1 = L.Wgrad(sw_feat, one.c(0), s_dh1, B, 1, 1, 1, fs, fs, L.dptr(st.view("2.weight", grad=True)), bnp, 1, 1, 1)
            dg1 = ops.make_conv(s_dh1, 1, one.c(1), B, (1, 1, 1), eng.packed_bwd["2"], self.dfeat, npass=bnp)
            self.keep += [s_dh2, wg2, dg2, s_dh1, wg1, dg1]
            self.wgrads += [wg2, wg1]
            bw.append(Launch(lib.coclr_conv_wgrad, (C.byref(wg2),), 1, AFTER0))
            bw.append(Launch(lib.coclr_conv_igemm, (C.byref(dg2), nsm)))
            bw.append(Launch(lib.coclr_bias_relu_bwd, (L.dptr(self.h1), L.dptr(b2), L.dptr(self.dh1),
                                                    L.dptr(st.view("2.bias", grad=True)), B, fs)))
            bw.append(split_op(self.dh1, self.dh1_pl, B, fs, None, None, False))
            bw.append(Launch(lib.coclr_conv_wgrad, (C.byref(wg1),), 1, AFTER0))
            bw.append(Launch(lib.coclr_conv_igemm, (C.byref(dg1), nsm)))
            bw.append(Launch(lib.coclr_avgpool_bwd, (L.dptr(self.dfeat), L.dptr(out.grad), out.spec.C, 0, B, Pn, fs)))
            grad_seen(out)
        elif g.pooled:
            self.dfeat = torch.empty(B, fs, dtype=torch.float32, device=dev)
            bw.append(Launch(lib.coclr_avgpool_bwd, (L.dptr(self.dfeat), L.dptr(out.grad), out.spec.C, 0, B, Pn, fs)))
            grad_seen(out)
        convs_into, pool_into = {}, {}
        for kind, it in g.items:
            if kind == "conv":
                convs_into.setdefault(it.dst.index, []).append(it)
            elif kind == "pool":
                pool_into[it.dst.index] = it
        # reverse forward order: a tensor is handled at its BatchNorm / pool item, i.e. after every consumer
        for kind_r, it_r in reversed(g.items):
            if kind_r == "conv":
                continue
            t = it_r if kind_r == "bn" else it_r.dst
            a = acts[t.index]
            if not a.grad_written:
                raise RuntimeError("tensor %s never receives a gradient" % t.name)
            if t.pending:
                if t.gates:
                    # a.grad holds d/d(gated output); turn it into d/d(un-gated activation) and emit the fc gradients
                    Pn = a.dims[0] * a.dims[1] * a.dims[2]
                    a.dgate = torch.empty(B, t.C, dtype=torch.float32, device=dev)
                    a.dmean = torch.empty(B, t.C, dtype=torch.float32, device=dev)
                    bw.append(Launch(lib.coclr_gate_bwd_reduce, (L.dptr(a.data), t.C, L.dptr(a.scale), L.dptr(a.shift),
                                                              t.relu, L.dptr(a.grad), t.C, B, Pn, t.C, L.dptr(a.dgate))))
                    for nm, coff, c in t.gates:
                        bw.append(Launch(lib.coclr_gate_fc_bwd, (L.dptr(a.dgate), L.dptr(a.gate), L.dptr(a.gmean),
                                                              L.dptr(st.view(nm + ".fc.weight")),
                                                              L.dptr(st.view(nm + ".fc.weight", grad=True)),
                                                              L.dptr(st.view(nm + ".fc.bias", grad=True)), L.dptr(a.dmean),
                                                              B, t.C, coff, c)))
                    bw.append(Launch(lib.coclr_gate_bwd_apply, (L.dptr(a.grad), t.C, L.dptr(a.gate), L.dptr(a.dmean), B, Pn,
                                                             t.C)))
                a.bsums = torch.zeros(2 * t.C, dtype=torch.float64, device=dev)
                a.bamax = torch.zeros(2 * t.C, dtype=torch.float32, device=dev)
                first = t.bn_members[0][0]
                goff = st.offsets[first + ".weight"][0]
                boff_b = st.offsets[first + ".bias"][0]
                if t.residual is not None:
                    ra = acts[t.residual.index]
                    res_args = (L.dptr(ra.pl.hi), L.dptr(ra.pl.lo), ra.pl.ld, 0, ra.pl.bf16,
                                L.dptr(ra.grad), ra.spec.C, 0, int(grad_seen(ra)))
                else:
                    res_args = (None, None, 0, 0, 0, None, 0, 0, 0)
                bb = L.BnBwd(L.dptr(a.data), L.dptr(a.grad), t.C, 0, t.C, a.M, L.dptr(a.scale), L.dptr(a.shift),
                             L.dptr(a.mean), L.dptr(a.rstd), t.relu, L.dptr(a.bsums),
                             L.dptr(st.grad[goff:]), L.dptr(st.grad[boff_b:]), L.dptr(a.dy.hi), L.dptr(a.dy.lo), *res_args,
                             0 if gbf else 1, L.dptr(a.bamax), L.dptr(a.dy_scale))
                oscale = None if gbf else a.dy_scale[1:]
                self.keep.append(bb)
                bw.append(Launch(lib.coclr_bn_bwd, (C.byref(bb), nsm)))
                for it in convs_into[t.index]:
                    sa = acts[it.src.index]
                    geom = ops.Geometry(it.k_eff, it.s_eff, it.p_eff)
                    dy = a.dy.src(it.dst_coff, _round8(it.cout), a.dims[0], a.dims[1], a.dims[2])
                    kreal = geom.taps * it.src_C
                    splits = 1   # one fp32 add per dW element: reproducible
                    wsrc = src_of(sa, it)
                    if it.s2d:
                        # the weight gradient is produced in the space-to-depth layout, then scattered back
                        dw_eff = eng.s2d[it.name]["dw_eff"]
                        wg = L.Wgrad(wsrc, geom.c(0), dy, B, a.dims[0], a.dims[1], a.dims[2], it.cout, it.cin_eff,
                                     L.dptr(dw_eff), bnp, gbf, gbf, splits, L.dptr(oscale))
                        self.keep += [wg, dy]
                        self.s2d_wgrads.append(wg)
                        # lane 0, where its torch zeroing and scatter run, so not wg_ws (lane 1 may be using it)
                        bw.append(Launch(eng._s2d_wgrad_op(it.name), (C.byref(wg),)))
                    else:
                        wg = L.Wgrad(wsrc, geom.c(0), dy, B, a.dims[0], a.dims[1], a.dims[2], it.cout, it.cin,
                                     L.dptr(st.view_span([n + ".weight" for n in it.weight_names], grad=True)), bnp, gbf, gbf,
                                     splits, L.dptr(oscale))
                        self.keep += [wg, dy]
                        self.wgrads.append(wg)
                        bw.append(Launch(lib.coclr_conv_wgrad, (C.byref(wg),), 1, AFTER0))
                    if it.need_dgrad:
                        dg = ops.make_conv(dy, gbf, geom.c(1), B, sa.dims, eng.packed_bwd[it.name], sa.grad, it.src_coff,
                                           accumulate=grad_seen(sa, it.src_coff, it.src_C), npass=bnp, out_scale=oscale)
                        self.keep.append(dg)
                        bw.append(Launch(lib.coclr_conv_igemm, (C.byref(dg), nsm)))
            elif t.index in pool_into:
                it = pool_into[t.index]
                sa = acts[it.src.index]
                geom = ops.Geometry(it.k, it.s, it.p)
                pl = L.Pool(None, None, it.src.C, 0, None, None, t.C, 0, None, None, L.dptr(a.idx), B, t.C,
                            sa.dims[0], sa.dims[1], sa.dims[2], a.dims[0], a.dims[1], a.dims[2], geom.c(0),
                            L.dptr(a.grad), L.dptr(sa.grad), int(grad_seen(sa)))
                self.keep.append(pl)
                bw.append(Launch(lib.coclr_maxpool_bwd, (C.byref(pl),)))
        # one workspace for the weight-gradient launches on lane 1 (they run one after the other): per-CTA partial sums
        # are written with plain stores and reduced by a second launch instead of fp32 atomics into dW
        need = max([int(lib.coclr_wgrad_ws_floats(C.byref(w))) for w in self.wgrads] + [0])
        self.wg_ws = None
        if need > 0:
            self.wg_ws = torch.empty(need, dtype=torch.float32, device=dev)
            for w in self.wgrads:
                w.ws, w.ws_floats = L.dptr(self.wg_ws).value, need
            for w in self.s2d_wgrads:
                n_own = int(lib.coclr_wgrad_ws_floats(C.byref(w)))
                if n_own > 0:
                    own = torch.empty(n_own, dtype=torch.float32, device=dev)
                    self.keep.append(own)
                    w.ws, w.ws_floats = L.dptr(own).value, n_own
        self.bwd_kernels = _count_kernels(bw)   # a weight gradient's count depends on the workspace it was given


class EncoderEngine:
    """Executes one encoder (see module docstring)."""

    profile = None  # set to a list to collect (fn name, args, start event, end event) per launch (bench / tuning only)

    def __init__(self, store, graph, precision="parity"):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % list(PRECISIONS))
        self.store, self.graph, self.precision = store, graph, precision
        self.plans = {}
        self.lanes = None   # the streams of lanes 1..3 (created at the first launch)
        dev = store.device
        # input of the modules' autograd nodes, so that their outputs require a gradient whatever the caller passes in
        self.anchor = torch.zeros(1, device=dev, requires_grad=True)
        fnp, fbf, bnp = PRECISIONS[precision]
        self.packed_fwd, self.packed_bwd, self._packs = {}, {}, []
        for kind, it in graph.items:
            if kind != "conv":
                continue
            taps = it.k_eff[0] * it.k_eff[1] * it.k_eff[2]
            w = store.view_span([n + ".weight" for n in it.weight_names])
            if it.s2d:
                w = self._make_s2d(it, w, dev)
            pf = ops.PackedWeights(it.cout, it.cin_eff, taps, it.src_C, 0, fbf, dev)
            self.packed_fwd[it.name] = pf
            self._packs.append((pf, w, False))
            if it.need_dgrad:
                pb = ops.PackedWeights(it.cout, it.cin, taps, _round8(it.cout), 1, 1 if fbf else 0, dev)   # format of dY
                self.packed_bwd[it.name] = pb
                self._packs.append((pb, w, True))
        if graph.head_dim is not None:
            fs, hd = graph.feature_size, graph.head_dim
            for nm, co in (("2", fs), ("4", hd)):
                w = store.view(nm + ".weight")
                pf = ops.PackedWeights(co, fs, 1, fs, 0, fbf, dev)
                pb = ops.PackedWeights(co, fs, 1, _round8(co), 1, 1, dev)
                self.packed_fwd[nm], self.packed_bwd[nm] = pf, pb
                self._packs += [(pf, w, False), (pb, w, True)]

    def _make_s2d(self, it, w, dev):
        """Index map of the space-to-depth stem: W'[o, (dy*2+dx)*Cin + c, t, ty, tx] = W[o, c, t, 2ty+dy-1, 2tx+dx-1]
        (zero when an index is -1).  Returns the persistent W' tensor that is re-derived before every packing."""
        cout, cin, kt = it.cout, it.cin, it.k[0]
        idx = torch.zeros(cout, 4 * cin, kt, 4, 4, dtype=torch.long)
        msk = torch.zeros(cout, 4 * cin, kt, 4, 4, dtype=torch.float32)
        o = torch.arange(cout).view(-1, 1)
        t = torch.arange(kt).view(1, -1)
        for dy in range(2):
            for dx in range(2):
                for ty in range(4):
                    for tx in range(4):
                        ky, kx = 2 * ty + dy - 1, 2 * tx + dx - 1
                        if ky < 0 or kx < 0:
                            continue
                        for c in range(cin):
                            idx[:, (dy * 2 + dx) * cin + c, :, ty, tx] = (((o * cin + c) * kt + t) * 7 + ky) * 7 + kx
                            msk[:, (dy * 2 + dx) * cin + c, :, ty, tx] = 1.0
        d = {"idx": idx.to(dev).view(-1), "mask": msk.to(dev).view(-1), "w": w,
             "w_eff": torch.zeros(cout, 4 * cin, kt, 4, 4, device=dev),
             "dw_eff": torch.zeros(cout, 4 * cin, kt, 4, 4, device=dev),
             "dw": self.store.view(it.name + ".weight", grad=True)}
        if not hasattr(self, "s2d"):
            self.s2d = {}
        self.s2d[it.name] = d
        return d["w_eff"]

    def _refresh_s2d(self):
        for d in getattr(self, "s2d", {}).values():
            torch.mul(d["w"].reshape(-1)[d["idx"]], d["mask"], out=d["w_eff"].view(-1))

    def _s2d_wgrad_op(self, name):
        """op(wg, stream): the weight gradient of the space-to-depth stem `name`; wg: byref of its coclr_wgrad_t."""
        d = self.s2d[name]
        lib = L.load()

        def op(wg, stream):
            d["dw_eff"].zero_()
            rc = lib.coclr_conv_wgrad(wg, stream)
            # W' -> W is one-to-one on the valid entries (masked entries point at index 0 with a zero factor)
            d["dw"].view(-1).index_add_(0, d["idx"], d["dw_eff"].view(-1) * d["mask"])
            return rc
        op.__name__ = "coclr_conv_wgrad_s2d"
        return op

    def _pack_table(self, backward):
        """Device table for coclr_pack_weights_batch (built once per variant: the pointers never change)."""
        key = bool(backward)
        tabs = getattr(self, "_pack_tables", None)
        if tabs is None:
            tabs = self._pack_tables = {}
        if key not in tabs:
            entries = [(pw, w) for pw, w, is_bwd in self._packs if backward or not is_bwd]
            arr = (L.Pack * len(entries))()
            starts = [0]
            for i, (pw, w) in enumerate(entries):
                assert w.is_contiguous() and w.dtype == torch.float32
                arr[i] = L.Pack(L.dptr(w), pw.Cout, pw.Cin, pw.taps, pw.cpad, pw.mode, pw.bf16,
                                L.dptr(pw.wpk), L.dptr(pw.unscale))
                starts.append(starts[-1] + pw.BN * pw.n_tiles)
            dev = self.store.device
            raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev) if not L.DRY_RUN else None
            rs = torch.tensor(starts, dtype=torch.int32, device=dev) if not L.DRY_RUN else None
            tabs[key] = (raw, rs, len(entries), starts[-1])
        return tabs[key]

    def pack_weights(self, backward=True):
        """Re-derive the 16-bit hi/lo tile images from the current fp32 weights (one launch for all layers)."""
        self._refresh_s2d()
        raw, rs, n, rows = self._pack_table(backward)
        L.check(L.load().coclr_pack_weights_batch(L.dptr(raw), L.dptr(rs), n, rows, L.stream_ptr()),
                "coclr_pack_weights_batch")

    def plan(self, B, T, H, W, training, with_backward, replica=0):
        """The plan of one input shape.  `replica` r > 0 gives a separate plan (own activations) of the same shape, so
        that the chunks of a data-parallel batch each keep theirs until backward; replica 0 is the plain shape key."""
        key = (B, T, H, W, bool(training), bool(with_backward))
        if replica:
            key += (int(replica),)
        p = self.plans.get(key)
        if p is None:
            p = Plan(self, B, T, H, W, training, with_backward)
            p.generation = 0   # training forwards that have filled the plan (see backward)
            self.plans[key] = p
        return p

    def _launch(self, records, kernels):
        """Launch a plan's Launch records and add their `kernels` to L.LAUNCHES.  Lane 0 is the current stream; before
        a launch, its lane waits for what the record's `wait` names, and lane 0 waits for every lane still open at the
        end.  Under `profile` every launch runs on lane 0 between two timing events."""
        main = torch.cuda.current_stream()
        if self.lanes is None:
            self.lanes = [torch.cuda.Stream() for _ in range(3)]
        lanes = [main] + self.lanes
        ptrs = [C.c_void_p(s.cuda_stream) for s in lanes]
        prof = EncoderEngine.profile
        fork, open_lanes = None, set()
        for r in records:
            lane = r.lane if prof is None else 0
            if prof is None and r.wait is not None:
                s = lanes[lane]
                if r.wait == FORK:
                    fork = torch.cuda.Event()
                    fork.record(main)
                if r.wait in (FORK, AT_FORK, AFTER1):
                    s.wait_event(fork)
                if r.wait in (AFTER1, AFTER0):
                    s.wait_stream(lanes[1 if r.wait == AFTER1 else 0])
                if r.wait == JOIN:
                    for ln in open_lanes:
                        main.wait_stream(lanes[ln])
                    open_lanes = set()
                else:
                    open_lanes.add(lane)
            if prof is not None:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
            rc = r.fn(*r.args, ptrs[lane])
            if prof is not None:
                e1.record()
                prof.append((r.fn.__name__, r.args, e0, e1))
            if rc != 0:
                raise L.CoclrError("%s failed with code %d" % (r.fn.__name__, rc))
        for ln in open_lanes:
            main.wait_stream(lanes[ln])
        L.LAUNCHES += kernels

    def forward(self, x, training=True, with_backward=False, repack=True, batch_index=None, batch=None, peers=None,
                norm=None, replica=0):
        """x: [*, C, T, H, W] fp32 CUDA (any batch stride). Clip b of the pass is x[batch_index[b]] when a
        device int64 index is given (shuffle-BN gather), else x[b].  peers = (device pointer of an array with one
        peer-mapped clip buffer per rank, clips per rank): batch_index then is a GLOBAL clip index and the clips are
        read straight from the owning ranks' buffers (same layout as x) over NVLink.  norm = (mean, std) device fp32
        [C]: per-channel (x - mean) / std applied while packing (the reference's GPU-side T.Normalize).  replica: plan
        slot (see plan()).  Only the three
        innermost dims of x must be dense: batch and channel strides are free, so a clip may be a view into the loader's
        [B, C, num_seq*seq_len, H, W] tensor.  Returns the plan; plan.q holds
        the normalised features [B, dim] (plan.backbone_out the backbone output when there is no head).  With
        with_backward, plan.generation right after the call is the token that backward() takes."""
        if not x.is_cuda:
            raise L.CoclrError("coclr_b200 encoders run on CUDA only (no CPU fallback)")
        _, Cin, T, H, W = x.shape
        B = x.shape[0] if batch is None else batch
        assert Cin == self.graph.first_channel and x.dtype == torch.float32
        assert x.stride(4) == 1 and x.stride(3) == W and x.stride(2) == H * W
        nm, ns = (L.dptr(norm[0]), L.dptr(norm[1])) if norm is not None else (None, None)
        if batch_index is not None:
            assert batch_index.dtype == torch.long and batch_index.is_cuda and batch_index.numel() == B
        p = self.plan(B, T, H, W, training, with_backward, replica)
        lib = L.load()
        peer_ptr, cpp = (C.c_void_p(int(peers[0])), int(peers[1])) if peers is not None else (None, 0)
        assert peers is None or batch_index is not None
        # the clip pointer / shuffle index change from call to call, so packing stays outside the captured graph
        if self.graph.stem_s2d:
            assert H % 2 == 0 and W % 2 == 0, "the space-to-depth stem needs even H, W"
            L.check(lib.coclr_pack_input_s2d(L.dptr(x), x.stride(0), x.stride(1), Cin, L.dptr(p.input.pl.hi),
                                             L.dptr(p.input.pl.lo), None, None, B, T, H, W, S2D_PAD,
                                             L.dptr(batch_index), peer_ptr, cpp, nm, ns, L.stream_ptr()),
                    "coclr_pack_input_s2d")
        else:
            L.check(lib.coclr_pack_input(L.dptr(x), x.stride(0), x.stride(1), Cin, L.dptr(p.input.pl.hi),
                                         L.dptr(p.input.pl.lo), None, None, B, T * H * W, L.dptr(batch_index),
                                         peer_ptr, cpp, nm, ns, L.stream_ptr()), "coclr_pack_input")

        def body():
            if repack:
                self.pack_weights(backward=with_backward)
            if training:
                p.stats.zero_()
                self.store.nbt += 1
            self._launch(p.fwd, p.fwd_kernels)
        self._graphed(p, "fwd" + ("_repack" if repack else ""), body, p.fwd_kernels + int(repack))   # + pack_weights
        if with_backward:
            p.generation += 1
        return p

    use_graphs = True   # capture every launch list into a CUDA graph after its first eager run

    def _graphed(self, p, key, body, kernels):
        """Every launch of `body` has fixed pointers and shapes: after one eager run (which also performs the
        one-time cudaFuncSetAttribute calls) capture it -- stream forks/joins included -- into a CUDA graph and
        replay that; the host then enqueues an encoder pass with one call instead of ~400.  kernels: the library
        kernels body launches, which a replay adds to L.LAUNCHES (an eager or captured run of body counts them)."""
        if not EncoderEngine.use_graphs or EncoderEngine.profile is not None:
            body()
            return
        state = p.graphs.get(key)
        if state is None:
            body()
            p.graphs[key] = "warm"
        elif state == "warm":
            g = p.graphs[key] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            g.replay()
        else:
            state.replay()
            L.LAUNCHES += kernels

    def backward(self, p, grad, generation):
        """grad: gradient w.r.t. the pass's output -- the normalised features [B, dim] with a head, the pooled feature
        [B, feature_size] of a `pooled` graph; accumulates into store.grad.  generation: plan.generation as forward()
        left it.  The plan's activations are shared by every pass of its shape, so a backward whose pass was
        overwritten by a later training forward raises."""
        if p.generation != generation:
            raise L.CoclrError("backward of an engine pass whose saved activations were overwritten by a later forward "
                               "of the same shape (one outstanding training forward per module and input shape)")
        (p.dq if self.graph.head_dim is not None else p.dfeat).copy_(grad)
        self._graphed(p, "bwd", lambda: self._launch(p.bwd, p.bwd_kernels), p.bwd_kernels)

    def backbone_output_ncdhw(self, p):
        return p.backbone_out.pl.value().permute(0, 4, 1, 2, 3).contiguous()
