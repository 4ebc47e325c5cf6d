"""LinearClassifier -- drop-in module surface of the reference's model/classifier.py (:10-69).

Same constructor, initialisation (fc N(0, 0.01), bias 0; final BN weight 1, bias 0), `forward(block) -> (logit, feat3d)`
and state_dict keys (`backbone.*` with the `blockN.i` aliases, `final_bn.*`, `final_fc.0.*` or `final_fc.1.*`), so
eval/main_classifier.py and reference checkpoints keep working.  The backbone runs as one engine pass that ends with
the average-pooled feature (coclr_b200.engine, `pooled` graph); F.normalize -> BatchNorm1d -> Dropout -> Linear run as
the classifier-head kernels of csrc/classifier.cu.  CUDA only: constructing on CPU is fine, calling forward on CPU
raises.

Every submodule's own `training` flag is honoured, as the reference's linear probe needs (`model.eval()` then
`final_bn.train()`, eval/main_classifier.py:319-325).  When no backbone parameter requires a gradient (or grad mode is
off) the backbone runs forward-only: no backward plan, and its parameters and, in eval mode, its running statistics are
left untouched.  With a trainable backbone the whole forward is one autograd node whose backward runs the head backward
and hands the pooled feature's gradient to the engine.  Parameter gradients are written into flat buffers (the
nn.Parameter .grad fields are views of them) and accumulate; `flat_spans()` exposes those buffers to
coclr_b200.moco.SpanAdam.  `feat3d` is returned without a gradient path.

The dropout mask comes from a counter-based Philox generator on the device, seeded from torch's default generator (so
`torch.manual_seed` makes runs reproducible); it is not bit-equal to torch's own dropout mask.  The mask of the last
forward is kept in `dropout_mask` ([B, feature_size] uint8, 1 = kept).

`replicas=R` (R > 1) makes forward() compute what nn.DataParallel(model, device_ids=<R GPUs>) computes (the reference's
multi-GPU fine-tuning and linear probe), on the model's one device.  The batch is split as torch.chunk(block, R) does
(`replica_chunks`), and wherever it is read as a batch -- a train-mode backbone, a train-mode final_bn -- each chunk
runs as its own pass: its own BatchNorm statistics and dropout seed.  As DataParallel's replica 0 shares the module's
buffers and the other replicas' updates are lost, the running statistics and num_batches_tracked end as chunk 0 left
them.  The outputs are the chunks' outputs concatenated; gradients accumulate over the chunks (DataParallel's
reduce-add).  A pass whose BatchNorms are all in eval mode reads no batch statistics and runs over all B clips at once,
and a frozen eval-mode backbone (the linear probe) runs once over B with only the head chunked.  infer() is always
one pass.  Every replica runs on the model's device (`_replica_device`).
"""
import ctypes as C

import torch
import torch.nn as nn

from backbone.select_backbone import select_backbone
from coclr_b200 import lib as L
from coclr_b200.engine import Graph, ParamStore, bind_engine


def replica_chunks(B, replicas):
    """Row ranges [(r0, r1)] of torch.chunk(x, replicas, dim=0) for a batch of B: ceil(B / replicas) rows each, the
    last one shorter; fewer than `replicas` chunks when B does not fill them (DataParallel then runs only that many)."""
    step = -(-B // replicas)
    return [(r0, min(r0 + step, B)) for r0 in range(0, B, step)]


class _ClassifierFn(torch.autograd.Function):
    """LinearClassifier._run as one autograd node.  Backward splits dlogits by chunk and runs each chunk's head backward
    and backbone backward in replica order; both accumulate into the flat gradients, which therefore end with the sum
    over the replicas."""

    @staticmethod
    def forward(ctx, anchor, model, x, chunks, backbone_grad):
        logits, feat3d, passes = model._run(x, chunks, backbone_grad, norm=model._input_norm(x.device))
        ctx.model, ctx.passes, ctx.backbone_grad = model, passes, backbone_grad
        ctx.mark_non_differentiable(feat3d)
        return logits, feat3d

    @staticmethod
    def backward(ctx, dlogits, _dfeat3d):
        model = ctx.model
        model._prepare_grads(ctx.backbone_grad)
        for plan, generation, heads in ctx.passes:
            for hd, (r0, r1) in heads:
                model._head_backward(hd, dlogits[r0:r1].contiguous(), ctx.backbone_grad)
            if ctx.backbone_grad:
                dfeat = heads[0][0]["dfeat"] if len(heads) == 1 else torch.cat([hd["dfeat"] for hd, _ in heads])
                model._engine.backward(plan, dfeat, generation)
        return None, None, None, None, None


class LinearClassifier(nn.Module):
    def __init__(self, num_class=101, network='resnet50', dropout=0.5, use_dropout=True, use_l2_norm=False,
                 use_final_bn=False, precision="parity", replicas=1):
        super().__init__()
        if int(replicas) < 1:
            raise ValueError("replicas must be >= 1, got %r" % (replicas,))
        self.replicas = int(replicas)
        self.network = network
        self.num_class = num_class
        self.dropout = dropout
        self.use_dropout = use_dropout
        self.use_l2_norm = use_l2_norm
        self.use_final_bn = use_final_bn
        self.precision = precision

        message = 'Classifier to %d classes with %s backbone;' % (num_class, network)
        if use_dropout:
            message += ' + dropout %f' % dropout
        if use_l2_norm:
            message += ' + L2Norm'
        if use_final_bn:
            message += ' + final BN'
        print(message)

        self.backbone, self.param = select_backbone(network)
        self.backbone.precision = precision

        if use_final_bn:
            self.final_bn = nn.BatchNorm1d(self.param['feature_size'])
            self.final_bn.weight.data.fill_(1)
            self.final_bn.bias.data.zero_()

        if use_dropout:
            self.final_fc = nn.Sequential(nn.Dropout(dropout), nn.Linear(self.param['feature_size'], self.num_class))
        else:
            self.final_fc = nn.Sequential(nn.Linear(self.param['feature_size'], self.num_class))
        self._initialize_weights(self.final_fc)
        self._engine = None
        self._head = None
        self.dropout_mask = None
        self._input_tf = None
        self._input_tf_dev = None

    def set_input_transform(self, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        """Fold the reference's GPU-side T.Normalize(mean, std, channel=1) (eval/main_classifier.py:216-220) into the
        engine's input packing: after this call forward() takes clips [B, 3, T, H, W] in [0, 1] (what ToTensor and
        coclr_b200.clf_augment give) and normalises them on the fly, with no extra pass.  mean=None switches it off
        (the default).  infer() is unaffected: it takes its `norm` argument."""
        self._input_tf = None if mean is None else (tuple(float(v) for v in mean), tuple(float(v) for v in std))
        self._input_tf_dev = None

    def _input_norm(self, device):
        if self._input_tf is None:
            return None
        if self._input_tf_dev is None or self._input_tf_dev[0].device != device:
            self._input_tf_dev = tuple(torch.tensor(v, dtype=torch.float32, device=device) for v in self._input_tf)
        return self._input_tf_dev

    def _initialize_weights(self, module):
        for name, param in module.named_parameters():
            if 'bias' in name:
                nn.init.constant_(param, 0.0)
            elif 'weight' in name:
                nn.init.normal_(param, mean=0.0, std=0.01)

    # -- flat storage ---------------------------------------------------------------------------------
    def _engine_for(self, device):
        bb = self.backbone
        self._engine = bind_engine(self._engine, bb.get_parameter(bb._probe), bb,
                                   lambda: Graph(bb._stages, bb.input_channel, feature_size=self.param['feature_size'],
                                                 pooled=True), self.precision)
        fc = "final_fc.%d." % (len(self.final_fc) - 1)
        if self._head is None or not self._head.owns(self.get_parameter(fc + "weight")):
            # one flat fp32 buffer (+ gradient) for the head parameters, names as in state_dict
            names = [fc + "weight", fc + "bias"] + (["final_bn.weight", "final_bn.bias"] if self.use_final_bn else [])
            named = {n: self.get_parameter(n) for n in names}
            self._head = ParamStore([(n, tuple(p.shape)) for n, p in named.items()], named[fc + "weight"].device)
            self._head.bind_module(named, {})
        return self._engine

    def flat_spans(self):
        """{'backbone': (params, grad), 'head': (params, grad)}: the flat fp32 buffers the parameters are views of."""
        eng = self._engine_for(self.final_fc[-1].weight.device)
        return {"backbone": (eng.store.flat, eng.store.grad), "head": (self._head.flat, self._head.grad)}

    def _prepare_grads(self, backbone):
        """(Re-)attach the .grad views of the head and, with `backbone`, of the backbone (ParamStore.attach_grads)."""
        if backbone:
            self._engine.store.attach_grads()
        self._head.attach_grads()

    # -- forward / backward -----------------------------------------------------------------------------
    def _replica_device(self, r):
        """Device of replica r: the model's own for every replica (one place to change for one GPU per replica)."""
        return self.final_fc[-1].weight.device

    def _running_state(self):
        """Every buffer a forward may update: the backbone's flat running statistics and num_batches_tracked, and
        final_bn's."""
        st = self._engine.store
        out = [st.running_mean, st.running_var, st.nbt]
        if self.use_final_bn:
            bn = self.final_bn
            out += [bn.running_mean, bn.running_var, bn.num_batches_tracked]
        return out

    def _run(self, block, chunks, backbone_grad, batch_index=None, batch=None, norm=None):
        """nn.DataParallel's forward over `chunks`, row ranges of the batch (see the module docstring; [(0, B)] is one
        plain pass).  Returns the gathered (logits, feat3d) and the passes for backward: [(plan, generation, [(head
        buffers, (r0, r1))])], one pass per chunk when the backbone is in train mode, else one pass over B with one
        head per chunk."""
        eng = self._engine_for(block.device)
        fs = self.param['feature_size']
        if self.use_final_bn and self.final_bn.training and any(r1 - r0 == 1 for r0, r1 in chunks):
            raise ValueError("Expected more than 1 value per channel when training, got input size %s" % ([1, fs],))
        for r in range(len(chunks)):
            if self._replica_device(r) != block.device:
                raise L.CoclrError("replica %d runs on %s, the input is on %s"
                                   % (r, self._replica_device(r), block.device))
        state = self._running_state() if len(chunks) > 1 else None
        kept = None
        passes, logits, feats, masks = [], [], [], []
        # a train-mode backbone reads its batch: one pass (own plan slot) per chunk; else one pass over all the clips
        groups = [[c] for c in chunks] if self.backbone.training else [chunks]
        for r, heads in enumerate(groups):
            x0 = heads[0][0]
            x = block if len(groups) == 1 else block[x0:heads[-1][1]]
            plan = eng.forward(x, training=self.backbone.training, with_backward=backbone_grad, repack=r == 0,
                               batch_index=batch_index, batch=batch, norm=norm, replica=r)
            hds = []
            for r0, r1 in heads:
                lg, hd = self._head_forward(plan.feat[r0 - x0:r1 - x0].clone())
                hds.append((hd, (r0, r1)))
                logits.append(lg)
                feats.append(hd.get("xn", hd["feat"]))
                masks.append(hd.get("mask"))
                if state is not None and kept is None:     # the running statistics end as chunk 0 left them
                    kept = [t.clone() for t in state]
            passes.append((plan, plan.generation, hds))
        if kept is not None:
            with torch.no_grad():
                for t, v in zip(state, kept):
                    t.copy_(v)
        if len(chunks) == 1:
            self.dropout_mask = masks[0]
            return logits[0], feats[0], passes
        self.dropout_mask = None if masks[0] is None else torch.cat(masks)
        return torch.cat(logits), torch.cat(feats), passes

    def _head_forward(self, feat):
        """Classifier-head forward (coclr_cls_head_fwd) of the pooled features feat [B, feature_size] (kept in the
        returned buffers); updates final_bn's running statistics in train mode.  Returns (logits, head buffers)."""
        B, fs = feat.shape
        f32 = dict(dtype=torch.float32, device=feat.device)
        hd = {"feat": feat}
        bn_train = self.use_final_bn and self.final_bn.training
        p = float(self.final_fc[0].p) if self.use_dropout else 0.0
        drop = self.use_dropout and self.final_fc[0].training and p > 0
        fc = self.final_fc[-1]
        h = L.ClsHead(B=B, fs=fs, ncls=fc.out_features, l2norm=int(self.use_l2_norm), bn=int(self.use_final_bn),
                      bn_training=int(bn_train), dropout=int(drop), p=p)
        h.feat, h.W, h.bias = L.dptr(hd["feat"]), L.dptr(fc.weight), L.dptr(fc.bias)
        if self.use_l2_norm:
            hd["xn"], hd["inv_norm"] = torch.empty(B, fs, **f32), torch.empty(B, **f32)
            h.xn, h.inv_norm = L.dptr(hd["xn"]), L.dptr(hd["inv_norm"])
        if self.use_final_bn:
            bn = self.final_bn
            hd["xb"], hd["mean"], hd["rstd"] = torch.empty(B, fs, **f32), torch.empty(fs, **f32), torch.empty(fs, **f32)
            h.xb, h.mean, h.rstd = L.dptr(hd["xb"]), L.dptr(hd["mean"]), L.dptr(hd["rstd"])
            h.gamma, h.beta = L.dptr(bn.weight), L.dptr(bn.bias)
            h.running_mean, h.running_var = L.dptr(bn.running_mean), L.dptr(bn.running_var)
            h.momentum, h.eps = bn.momentum, bn.eps
        if drop:
            hd["mask"] = torch.empty(B, fs, dtype=torch.uint8, device=feat.device)
            hd["xd"] = torch.empty(B, fs, **f32)
            h.mask, h.xd = L.dptr(hd["mask"]), L.dptr(hd["xd"])
            h.seed = int(torch.randint(0, 2 ** 62, (1,)))     # torch's default generator: torch.manual_seed applies
        logits = torch.empty(B, fc.out_features, **f32)
        h.logits = L.dptr(logits)
        L.check(L.load().coclr_cls_head_fwd(C.byref(h), L.stream_ptr()), "coclr_cls_head_fwd")
        if bn_train:
            self.final_bn.num_batches_tracked.add_(1)
        hd["struct"] = h
        return logits, hd

    def _head_backward(self, hd, dlogits, backbone_grad):
        h = hd["struct"]
        B, fs = h.B, h.fs
        gv = [self._head.view(n, grad=True) for n in self._head.offsets]
        hd["dx"] = torch.empty(B, fs, dtype=torch.float32, device=dlogits.device)
        hd["dfeat"] = torch.empty(B, fs, dtype=torch.float32, device=dlogits.device) if backbone_grad else None
        h.dlogits, h.dx, h.dfeat = L.dptr(dlogits), L.dptr(hd["dx"]), L.dptr(hd["dfeat"])
        h.dW, h.dbias = L.dptr(gv[0]), L.dptr(gv[1])
        if self.use_final_bn:
            h.dgamma, h.dbeta = L.dptr(gv[2]), L.dptr(gv[3])
        L.check(L.load().coclr_cls_head_bwd(C.byref(h), L.stream_ptr()), "coclr_cls_head_bwd")

    def forward(self, block):
        """block [B, C, T, H, W] -> (logit [B, num_class], feat3d [B, feature_size]) (classifier.py:47-61)."""
        if not block.is_cuda:
            raise L.CoclrError("coclr_b200 classifiers run on CUDA (sm_90a) only; there is no CPU path")
        eng = self._engine_for(block.device)
        grad_on = torch.is_grad_enabled()
        backbone_grad = grad_on and any(p.requires_grad for p in self.backbone.parameters())
        head_grad = grad_on and any(p.requires_grad for _, p in self._head.params)
        B = block.shape[0]
        batch_read = self.backbone.training or (self.use_final_bn and self.final_bn.training)
        chunks = replica_chunks(B, self.replicas) if self.replicas > 1 and batch_read else [(0, B)]
        if backbone_grad or head_grad:
            return _ClassifierFn.apply(eng.anchor, self, block, chunks, backbone_grad)
        with torch.no_grad():
            logits, feat3d, _ = self._run(block, chunks, False, norm=self._input_norm(block.device))
        return logits, feat3d

    @torch.no_grad()
    def infer(self, x, batch_index=None, batch=None, norm=None):
        """Inference only (no autograd node, no backward plan): (logit, feat3d) of the clips
        x[batch_index[b]] (b < batch; x[b] without an index), as forward() would return for them.  x is
        [*, C, T, H, W] with free batch and channel strides (a strided view into a larger buffer is fine);
        norm = (mean, std) device fp32 [C] applies the per-channel (x - mean) / std while the engine packs the input.
        Each submodule's `training` flag is honoured as in forward()."""
        if not x.is_cuda:
            raise L.CoclrError("coclr_b200 classifiers run on CUDA (sm_90a) only; there is no CPU path")
        B = x.shape[0] if batch is None else batch
        logits, feat3d, _ = self._run(x, [(0, B)], False, batch_index=batch_index, batch=batch, norm=norm)
        return logits, feat3d
