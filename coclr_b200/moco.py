"""Host-side pieces of the MoCo step shared by InfoNCE / UberNCE / CoCLR (model/pretrain.py):

* MoCoEncoder   -- nn.Sequential(backbone, avgpool, conv, relu, conv) with the reference's child indices
                   (model/pretrain.py:49-54) whose forward/backward run as one engine pass;
* nce_logits    -- autograd op: fused [q.k, q.queue]/T (+ cross-entropy by-products);
* nce_cross_entropy -- nn.CrossEntropyLoss-compatible criterion that reuses those by-products;
* momentum_update / enqueue / concat_all_gather helpers;
* FlatAdam      -- torch.optim.Adam semantics (main_nce.py:190-200) as one fused launch over the flat buffer.
"""
import ctypes as C
import math

import torch
import torch.distributed as dist
import torch.nn as nn

from . import lib as L
from .engine import Graph, ParamStore, EncoderEngine
from .s3d_spec import S3D_FEATURE_SIZE


# Per-phase timeline of a step (bench.py --timeline): CUDA events on whatever stream the phase runs on; off by default.
TIMELINE = None


def mark(name):
    if TIMELINE is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        TIMELINE.append((name, ev))


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


@torch.no_grad()
def concat_all_gather(tensor):
    """all_gather + cat(dim 0), no gradient (model/pretrain.py:14-25). World size 1 needs no process group."""
    world, _ = _world()
    if world == 1:
        return tensor
    out = torch.empty((world * tensor.shape[0],) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    dist.all_gather_into_tensor(out, tensor.contiguous())
    return out


class PeerClips:
    """Key clips of every rank, readable from every rank: two symmetric-memory staging buffers (NVLink peer-mapped via
    torch.distributed._symmetric_memory) per rank.  publish() copies the local clips in and runs a device-side
    barrier on the current stream; afterwards any rank may read any rank's clips with plain loads (the packing
    kernel does, coclr_pack_input*), so the all-gather of all clips (model/pretrain.py:105-106: W x 201 MB received
    per rank) shrinks to P2P reads of the B clips a rank actually encodes.  Double buffering makes the next
    publish() safe without a second barrier: a rank overwrites buffer i two steps later, after the barrier of the
    step in between, which every peer only passes once its reads of buffer i have been queued before it."""

    def __init__(self, shape, device, group):
        import torch.distributed._symmetric_memory as symm
        self.bufs = [symm.empty(*shape, dtype=torch.float32, device=device) for _ in range(2)]
        self.hdls = [symm.rendezvous(b, group) for b in self.bufs]
        self.cur = 0

    def publish(self, x):
        buf, hdl = self.bufs[self.cur], self.hdls[self.cur]
        self.cur ^= 1
        buf.copy_(x)
        hdl.barrier()
        return buf, hdl.buffer_ptrs_dev


class _EncodeFn(torch.autograd.Function):
    """Encoder pass as one autograd node; the parameter gradients are written straight into the
    encoder's flat gradient buffer (the nn.Parameter .grad fields are views of it)."""

    @staticmethod
    def forward(ctx, anchor, enc, x, training):
        plan = enc._engine_for(x.device).forward(x, training=training, with_backward=True, norm=enc.input_norm)
        # the plan (activation buffers + captured graphs) is shared by every pass of this shape: remember which pass
        # filled it, so that a backward whose activations were overwritten by a later forward fails loudly
        plan.generation = getattr(plan, "generation", 0) + 1
        ctx.enc, ctx.plan, ctx.generation = enc, plan, plan.generation
        return plan.q.clone()

    @staticmethod
    def backward(ctx, dq):
        enc = ctx.enc
        if ctx.plan.generation != ctx.generation:
            raise L.CoclrError("backward of an encoder pass whose saved activations were overwritten by a later forward "
                               "of the same shape (one outstanding training forward per encoder and input shape)")
        enc._prepare_grads()
        mark("bwd:start")
        enc._engine.backward(ctx.plan, dq.contiguous())
        mark("bwd:end")
        return None, None, None, None


class MoCoEncoder(nn.Sequential):
    """backbone + AdaptiveAvgPool3d + Conv3d(fs,fs,1) + ReLU + Conv3d(fs,dim,1); state_dict keys
    '0.<backbone>', '2.weight', '2.bias', '4.weight', '4.bias' as in the reference."""

    def __init__(self, backbone, feature_size, dim, precision="parity"):
        super().__init__(backbone,
                         nn.AdaptiveAvgPool3d((1, 1, 1)),
                         nn.Conv3d(feature_size, feature_size, kernel_size=1, bias=True),
                         nn.ReLU(),
                         nn.Conv3d(feature_size, dim, kernel_size=1, bias=True))
        self.feature_size, self.dim, self.precision = feature_size, dim, precision
        self._engine = None
        self._anchor = None
        self.input_norm = None   # (mean, std) device tensors: per-channel normalisation fused into the clip packing

    # -- engine -------------------------------------------------------------------------------
    def _engine_for(self, device):
        w = self[2].weight
        if not w.is_cuda:
            raise L.CoclrError("coclr_b200 encoders run on CUDA (sm_90a) only; there is no CPU path")
        e = self._engine
        if e is None or e.store.device != w.device or w.data_ptr() != e.store.view("2.weight").data_ptr():
            bb = self[0]
            graph = Graph(bb._stages, bb.input_channel, head_dim=self.dim, feature_size=self.feature_size,
                          bb_prefix="0.")
            store = ParamStore(graph, w.device)
            store.bind_module(dict(self.named_parameters()), dict(self.named_buffers()))
            self._engine = EncoderEngine(store, graph, self.precision)
            self._anchor = torch.zeros(1, device=w.device, requires_grad=True)
        return self._engine

    @property
    def store(self):
        return self._engine_for(self[2].weight.device).store

    def _prepare_grads(self):
        """(Re-)attach the .grad views; a parameter whose grad was set to None means 'zeroed'."""
        st = self._engine.store
        first = self[2].weight
        if first.grad is None or first.grad.data_ptr() != st.view("2.weight", grad=True).data_ptr():
            st.grad.zero_()
            st.attach_grads(dict(self.named_parameters()))

    def encode(self, x, batch_index=None, batch=None, peers=None):
        """L2-normalised features [B, dim] of clips x[B,C,T,H,W] (what the reference obtains with
        F.normalize(encoder(x), dim=1).view(B, dim); model/pretrain.py:153-155,165-167)."""
        eng = self._engine_for(x.device)
        want_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if want_grad:
            assert batch_index is None
            return _EncodeFn.apply(self._anchor, self, x, self.training)
        plan = eng.forward(x, training=self.training, with_backward=False, batch_index=batch_index, batch=batch,
                           peers=peers, norm=self.input_norm)
        return plan.q.clone()

    def forward(self, x):
        """Un-normalised projection [B, dim, 1, 1, 1] (the reference's `encoder(x)`); forward only."""
        eng = self._engine_for(x.device)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise L.CoclrError("use .encode() (autograd-aware) for training; forward() is inference-only")
        plan = eng.forward(x, training=self.training, with_backward=False, norm=self.input_norm)
        return (plan.h2.view(x.shape[0], self.dim) + self[4].bias).view(x.shape[0], self.dim, 1, 1, 1)


@torch.no_grad()
def momentum_update(enc_q, enc_k, m):
    """k = k*m + q*(1-m) over all parameters in one launch (model/pretrain.py:76-80)."""
    sq, sk = enc_q.store, enc_k.store
    assert sq.numel == sk.numel
    lib = L.load()
    m32 = float(torch.tensor(m, dtype=torch.float32))
    omm32 = float(torch.tensor(1. - m, dtype=torch.float32))
    L.check(lib.coclr_ema_update(L.dptr(sk.flat), L.dptr(sq.flat), m32, omm32, sk.numel, L.num_sms(sk.device),
                                 L.stream_ptr()), "coclr_ema_update")


@torch.no_grad()
def enqueue(queue, keys, ptr):
    """queue[:, ptr:ptr+n] = keys.T (model/pretrain.py:93)."""
    dim, K = queue.shape
    n = keys.shape[0]
    assert keys.shape[1] == dim and keys.is_contiguous() and queue.is_contiguous()
    L.check(L.load().coclr_queue_enqueue(L.dptr(queue), L.dptr(keys), dim, K, int(ptr), n, L.stream_ptr()),
            "coclr_queue_enqueue")


@torch.no_grad()
def mask_topk(kf, queue_second, k_vsource, queue_vname, topk):
    """CoCLR's positive mask [B, 1+K] bool (model/pretrain.py:392-413): column 0 and the same-source columns, plus --
    when topk > 0 -- the top-k columns of kf @ queue_second among the others."""
    B, K = k_vsource.shape[0], queue_vname.shape[0]
    assert k_vsource.dtype == torch.long and queue_vname.dtype == torch.long
    mask = torch.empty(B, K + 1, dtype=torch.bool, device=k_vsource.device)
    kf = kf.contiguous()
    assert queue_second.is_contiguous() and kf.shape[1] == queue_second.shape[0]
    L.check(L.load().coclr_mask_topk(L.dptr(kf), L.dptr(queue_second), L.dptr(k_vsource.contiguous()),
                                     L.dptr(queue_vname), B, kf.shape[1], K, int(topk), L.dptr(mask), L.stream_ptr()),
            "coclr_mask_topk")
    return mask


class _NCELogitsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, queue, T):
        B, D = q.shape
        K = queue.shape[1]
        q, k = q.contiguous(), k.contiguous()
        logits = torch.empty(B, K + 1, dtype=torch.float32, device=q.device)
        loss_rows = torch.empty(B, dtype=torch.float32, device=q.device)
        dlogits = torch.empty(B, K + 1, dtype=torch.float32, device=q.device)
        ws = torch.empty(2 * B * ((K + 1023) // 1024), dtype=torch.float32, device=q.device) if K > 2048 else None
        L.check(L.load().coclr_nce_logits_ce(L.dptr(q), L.dptr(k), L.dptr(queue), float(T), B, D, K, L.dptr(logits),
                                             L.dptr(loss_rows), L.dptr(dlogits), L.dptr(ws), L.stream_ptr()),
                "coclr_nce_logits_ce")
        # the queue is overwritten by the enqueue right after (pretrain.py:188); backward needs the old one
        ctx.save_for_backward(k, queue.clone())
        ctx.T, ctx.shape = float(T), (B, D, K)
        ctx.mark_non_differentiable(loss_rows, dlogits)
        return logits, loss_rows, dlogits

    @staticmethod
    def backward(ctx, dlogits, _a, _b):
        k, queue = ctx.saved_tensors
        B, D, K = ctx.shape
        dq = torch.empty(B, D, dtype=torch.float32, device=k.device)
        L.check(L.load().coclr_nce_logits_bwd(L.dptr(dlogits.contiguous()), L.dptr(k), L.dptr(queue), ctx.T, B, D, K,
                                              L.dptr(dq), L.stream_ptr()), "coclr_nce_logits_bwd")
        return dq, None, None, None


def nce_logits(q, k, queue, T):
    """logits [B, 1+K] = cat(q.k, q @ queue) / T (model/pretrain.py:175-182). The returned tensor carries
    the fused cross-entropy by-products for nce_cross_entropy()."""
    logits, loss_rows, dlogits = _NCELogitsFn.apply(q, k, queue, T)
    logits._coclr_ce = (loss_rows, dlogits)
    return logits


class _FusedCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, loss_rows, dlogits):
        ctx.save_for_backward(dlogits)
        return loss_rows.mean()

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None


def nce_cross_entropy(logits, labels=None):
    """nn.CrossEntropyLoss()(logits, labels) for labels == 0 (main_nce.py:201,314). When `logits` comes from
    nce_logits() the loss and its gradient were already produced by the fused kernel."""
    ce = getattr(logits, "_coclr_ce", None)
    if ce is not None:
        return _FusedCEFn.apply(logits, ce[0], ce[1])
    return torch.nn.functional.cross_entropy(logits, labels)


class FlatAdam:
    """torch.optim.Adam(lr, betas, eps, weight_decay) with coupled L2 over the flat parameter buffer of one
    MoCoEncoder (main_nce.py:190-200 builds one param group per tensor with identical hyper-parameters,
    which is equivalent). Gradients are all-reduced (mean) over the process group first (DDP, :172)."""

    def __init__(self, encoder, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5):
        self.encoder = encoder
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]
        self.step_count = 0
        self.exp_avg = self.exp_avg_sq = None

    def _state(self):
        st = self.encoder.store
        if self.exp_avg is None or self.exp_avg.device != st.flat.device:
            self.exp_avg = torch.zeros_like(st.flat)
            self.exp_avg_sq = torch.zeros_like(st.flat)
        return st

    def zero_grad(self, set_to_none=False):
        self._state().grad.zero_()

    @torch.no_grad()
    def step(self):
        st = self._state()
        world, _ = _world()
        mark("opt:allreduce_wait")
        if world > 1:
            dist.all_reduce(st.grad)
        mark("opt:allreduce_done")
        g = self.param_groups[0]
        self.step_count += 1
        b1, b2 = g["betas"]
        bc1 = 1.0 - b1 ** self.step_count
        bc2 = 1.0 - b2 ** self.step_count
        p = L.Adam(L.dptr(st.flat), L.dptr(st.grad), L.dptr(self.exp_avg), L.dptr(self.exp_avg_sq), st.numel,
                   1.0 / world, b1, b2, g["eps"], g["weight_decay"], g["lr"] / bc1, math.sqrt(bc2))
        L.check(L.load().coclr_adam_step(C.byref(p), L.num_sms(st.flat.device), L.stream_ptr()), "coclr_adam_step")
        mark("opt:adam_done")

    def state_dict(self):
        return {"step": self.step_count, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq,
                "param_groups": self.param_groups}

    def load_state_dict(self, sd):
        self.step_count = sd["step"]
        self.exp_avg, self.exp_avg_sq = sd["exp_avg"], sd["exp_avg_sq"]
        self.param_groups = sd["param_groups"]
