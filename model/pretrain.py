"""InfoNCE / UberNCE / CoCLR -- drop-in module surface of the reference's model/pretrain.py.

Same constructors, forward signatures, return values, buffers (`queue`, `queue_ptr`, `queue_label`,
`queue_second`, `queue_vname`) and state_dict key names as TengdaHan/CoCLR model/pretrain.py:28-418, so
main_nce.py / main_coclr.py and reference checkpoints keep working; the arithmetic runs on coclr_b200's
sm_90a kernels (CUDA only -- constructing on CPU is fine, calling forward on CPU raises).

What changed under the surface (see DESIGN.md):
  * encoders run as fused engine passes (coclr_b200.engine), BN/ReLU folded into the convs;
  * the momentum update is one launch over a flat buffer (reference: 705 launches, pretrain.py:76-80);
  * shuffle-BN keeps the reference's permutation semantics (rank 0 draws torch.randperm on the CPU RNG and
    broadcasts, :112-115) but the local pick x_gather[idx_this] is folded into the clip-packing kernel, and
    the un-shuffle all-gather (:133-143) and the enqueue all-gather (:85) are ONE all-gather;
  * logits + temperature + cross-entropy by-products come from one kernel (:175-182);
  * queue_ptr is mirrored on the host, so there is no `int(self.queue_ptr)` device sync per step (:89).
"""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.distributed as dist

from backbone.select_backbone import select_backbone
from coclr_b200 import moco
from coclr_b200.moco import concat_all_gather  # noqa: F401  (re-exported: reference defines it here)


class InfoNCE(nn.Module):
    """MoCo for video (reference model/pretrain.py:28-190)."""

    overlap_key_branch = True   # run EMA + shuffle + encoder_k on a side stream next to the query forward

    def __init__(self, network='s3d', dim=128, K=2048, m=0.999, T=0.07, precision="parity"):
        super().__init__()
        self.dim, self.K, self.m, self.T = dim, K, m, T
        self.precision = precision

        backbone, self.param = select_backbone(network)
        feature_size = self.param['feature_size']
        backbone.precision = precision
        self.encoder_q = moco.MoCoEncoder(backbone, feature_size, dim, precision)
        backbone, _ = select_backbone(network)
        backbone.precision = precision
        self.encoder_k = moco.MoCoEncoder(backbone, feature_size, dim, precision)
        for param_q, param_k in zip(self.encoder_q.parameters(), self.encoder_k.parameters()):
            param_k.data.copy_(param_q.data)      # initialise (pretrain.py:64-66)
            param_k.requires_grad = False         # not updated by gradient

        self.register_buffer("queue", nn.functional.normalize(torch.randn(dim, K), dim=0))
        self.register_buffer("queue_ptr", torch.zeros(1, dtype=torch.long))
        self._ptr_host = None
        self._side_stream = None
        self._peer_clips = {}     # clip shape -> moco.PeerClips, or False when symmetric memory is unavailable

    @property
    def module(self):
        """The reference's scripts reach the model through its DistributedDataParallel wrapper (`model.module.sampler`,
        `model.module.queue_is_full`, main_coclr.py:363,403).  There is no wrapper here (the flat gradient is all-reduced
        in FlatAdam.step), so `.module` is the model itself and those call sites keep working."""
        return self

    # -- fused input transform -----------------------------------------------------------------------
    def set_input_transform(self, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        """Fold the reference's GPU-side `tr` (main_nce.py:207-209,299-302: T.Normalize(mean, std, channel=1) ->
        view(B,3,num_seq,seq_len,H,W) -> transpose(1,2) -> contiguous) into the clip-packing kernel.  After this call
        forward() also accepts the loader's tensor as is -- [B, 3, num_seq*seq_len, H, W] in [0, 1] -- and every encoder
        normalises on the fly; the [B, 2, 3, T, H, W] form is normalised the same way.  mean=None switches it off."""
        self._input_tf = None if mean is None else (tuple(float(v) for v in mean), tuple(float(v) for v in std))
        self._input_tf_dev = None
        for enc in self._encoders():
            enc.input_norm = None

    def _encoders(self):
        return [m for m in (self.encoder_q, self.encoder_k, getattr(self, "sampler", None)) if m is not None]

    def _views(self, block):
        """The two clips of a sample as [B, C, T, H, W] views (no copies): from [B, 2, C, T, H, W] (what the reference's
        forward takes, pretrain.py:145-150) or from the loader layout [B, C, 2*T, H, W] (before `tr`)."""
        tf = getattr(self, "_input_tf", None)
        if tf is not None and getattr(self, "_input_tf_dev", None) is None:
            self._input_tf_dev = (torch.tensor(tf[0], dtype=torch.float32, device=block.device),
                                  torch.tensor(tf[1], dtype=torch.float32, device=block.device))
            for enc in self._encoders():
                enc.input_norm = self._input_tf_dev
        if block.dim() == 5:
            assert block.shape[2] % 2 == 0, "loader layout [B, C, 2*T, H, W] expected"
            T = block.shape[2] // 2
            return block[:, :, :T], block[:, :, T:]
        assert block.shape[1] == 2                                                    # pretrain.py:148
        return block[:, 0], block[:, 1]

    def load_state_dict(self, state_dict, *args, **kwargs):
        """Checkpoints written by the reference carry the DistributedDataParallel prefix (`module.encoder_q...`,
        main_nce.py:172,271-279; the published pretrained files do): accepted as is."""
        if any(k.startswith("module.") for k in state_dict):
            state_dict = type(state_dict)((k[len("module."):] if k.startswith("module.") else k, v)
                                          for k, v in state_dict.items())
        return super().load_state_dict(state_dict, *args, **kwargs)

    # -- queue pointer mirror ---------------------------------------------------------------------
    def _load_from_state_dict(self, *args, **kwargs):
        self._ptr_host = None  # re-read the loaded pointer lazily
        return super()._load_from_state_dict(*args, **kwargs)

    def _ptr(self):
        if self._ptr_host is None:
            self._ptr_host = int(self.queue_ptr)   # one sync after construction / load, not per step
        return self._ptr_host

    def _advance_ptr(self, n):
        self._ptr_host = (self._ptr() + n) % self.K
        self.queue_ptr.fill_(self._ptr_host)

    # -- pieces of the step --------------------------------------------------------------------------
    @torch.no_grad()
    def _momentum_update_key_encoder(self):
        moco.momentum_update(self.encoder_q, self.encoder_k, self.m)

    @torch.no_grad()
    def _shuffled_keys(self, x2, encoder=None):
        """shuffle-BN (pretrain.py:98-143): returns (k_local [B, dim], k_global [B*W, dim]) in the ORIGINAL
        (un-shuffled) order; k_global is what _dequeue_and_enqueue's all-gather (:85) would produce."""
        encoder = self.encoder_k if encoder is None else encoder
        world, rank = moco._world()
        B = x2.shape[0]
        peer = self._peer_exchange(x2) if world > 1 else None
        moco.mark("key:start")
        if peer is None:
            x_gather = concat_all_gather(x2) if world > 1 else x2                     # :105-106
        else:
            x_gather, peer_ptrs = peer.publish(x2)      # own clips; the other ranks' are read in place over NVLink
        moco.mark("key:clips_published")
        # CPU RNG draw as in the reference (:112); staged through pinned memory so that the host does not block on the copy
        if getattr(self, "_perm_pinned", None) is None or self._perm_pinned[0].numel() != B * world:
            self._perm_pinned = [torch.empty(B * world, dtype=torch.long) for _ in range(2)]
            if x2.is_cuda:
                self._perm_pinned = [t.pin_memory() for t in self._perm_pinned]
            self._perm_flip = 0
        pinned = self._perm_pinned[self._perm_flip]
        self._perm_flip ^= 1
        torch.randperm(B * world, out=pinned)
        idx_shuffle = torch.empty(B * world, dtype=torch.long, device=x2.device)
        idx_shuffle.copy_(pinned, non_blocking=True)
        if world > 1:
            dist.broadcast(idx_shuffle, src=0)                                       # :115
        moco.mark("key:perm_broadcast")
        idx_unshuffle = torch.argsort(idx_shuffle)
        idx_this = idx_shuffle.view(world, -1)[rank].contiguous()
        k_sh = encoder.encode(x_gather, batch_index=idx_this, batch=B,            # x_gather[idx_this], :124
                              peers=(peer_ptrs, B) if peer is not None else None)
        moco.mark("key:encoded")
        k_all = concat_all_gather(k_sh) if world > 1 else k_sh
        k_global = k_all[idx_unshuffle].contiguous()                                  # :143 for every rank
        moco.mark("key:gathered")
        return k_global[rank * B:(rank + 1) * B], k_global

    peer_shuffle = os.environ.get("COCLR_PEER_SHUFFLE", "1") != "0"

    def _peer_exchange(self, x2):
        """PeerClips for this clip shape, or None (-> all-gather path) when peer memory cannot be set up (no NVLink /
        P2P between the ranks, non-NCCL backend) or is switched off with COCLR_PEER_SHUFFLE=0."""
        if not InfoNCE.peer_shuffle or not x2.is_cuda or dist.get_backend() != "nccl":
            return None
        key = tuple(x2.shape)
        pc = self._peer_clips.get(key)
        if pc is None:
            ok = torch.ones(1, device=x2.device)
            try:
                pc = moco.PeerClips(key, x2.device, dist.group.WORLD)
            except Exception as ex:  # pragma: no cover - depends on the machine
                print("coclr_b200: peer-memory key exchange unavailable (%r); using all-gather" % (ex,))
                pc, ok[0] = False, 0
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)       # all ranks take the same path
            if float(ok) < 1:
                pc = False
            self._peer_clips[key] = pc
        return pc or None

    @torch.no_grad()
    def _dequeue_and_enqueue(self, keys_global):
        n = keys_global.shape[0]
        assert self.K % n == 0                                                        # pretrain.py:90
        ptr = self._ptr()
        moco.enqueue(self.queue, keys_global, ptr)
        self._advance_ptr(n)
        return ptr

    def _qk(self, block):
        if not block.is_cuda:
            raise moco.L.CoclrError("coclr_b200 modules run on CUDA (sm_90a) only; there is no CPU path")
        x1, x2 = self._views(block)                # views; the .contiguous() copies are folded into packing
        in_train_mode = torch.is_grad_enabled() and any(p.requires_grad for p in self.encoder_q.parameters())  # :157
        # the key branch (EMA -> shuffle -> encoder_k) does not depend on the query forward: run it on a side stream
        # so that the many small layers of the two encoders fill the SMs together
        main = torch.cuda.current_stream()
        if self._side_stream is None:
            # high priority: the key branch carries the cross-rank exchange (clip publish, barrier, permutation broadcast,
            # NVLink reads); when it gets the SMs first, that latency is covered by the query forward on the main stream
            # instead of sticking out behind it
            self._side_stream = torch.cuda.Stream(priority=-1)
        side = self._side_stream if InfoNCE.overlap_key_branch else main
        side.wait_stream(main)
        overlap = side is not main
        if overlap:
            # the query forward is enqueued FIRST: the key branch has host-side work (permutation draw, collectives) that
            # would otherwise keep the main stream idle for the first ~1 ms of the step
            moco.mark("query:start")
            q = self.encoder_q.encode(x1)                                             # :153-155
            moco.mark("query:encoded")
        with torch.cuda.stream(side), torch.no_grad():
            if in_train_mode:
                self._momentum_update_key_encoder()                                   # :161
            k, k_global = self._shuffled_keys(x2)
        if not overlap:
            moco.mark("query:start")
            q = self.encoder_q.encode(x1)                                             # :153-155
            moco.mark("query:encoded")
        main.wait_stream(side)
        moco.mark("joined")
        return q, k, k_global, in_train_mode

    def forward(self, block):
        """block [B,2,C,T,H,W] -> (logits [B,1+K] already / T, labels [B] zeros) (pretrain.py:145-190)."""
        q, k, k_global, in_train_mode = self._qk(block)
        logits = moco.nce_logits(q, k, self.queue, self.T)                            # :175-182
        labels = torch.zeros(logits.shape[0], dtype=torch.long, device=logits.device)  # :185
        if in_train_mode:
            self._dequeue_and_enqueue(k_global)                                       # :188
        return logits, labels


class UberNCE(InfoNCE):
    """Supervised InfoNCE: labels define the positives (reference model/pretrain.py:193-278)."""

    def __init__(self, network='s3d', dim=128, K=2048, m=0.999, T=0.07, precision="parity"):
        super().__init__(network, dim, K, m, T, precision)
        self.register_buffer("queue_label", torch.ones(K, dtype=torch.long) * -1)

    def forward(self, block, k_label):
        q, k, k_global, in_train_mode = self._qk(block)
        logits = moco.nce_logits(q, k, self.queue, self.T)
        mask = k_label.unsqueeze(1) == self.queue_label.unsqueeze(0)                  # :271
        mask = torch.cat([torch.ones((mask.shape[0], 1), dtype=torch.bool, device=mask.device), mask], dim=1)
        if in_train_mode:
            with torch.no_grad():
                labels_global = concat_all_gather(k_label)                            # :215
                ptr = self._dequeue_and_enqueue(k_global)
                self.queue_label[ptr:ptr + labels_global.shape[0]] = labels_global    # :224
        return logits, mask


class CoCLR(InfoNCE):
    """Co-training with a frozen second-view sampler (reference model/pretrain.py:281-418)."""

    def __init__(self, network='s3d', dim=128, K=2048, m=0.999, T=0.07, topk=5, reverse=False, precision="parity"):
        super().__init__(network, dim, K, m, T, precision)
        self.topk = topk
        backbone, _ = select_backbone(network)
        backbone.precision = precision
        self.sampler = moco.MoCoEncoder(backbone, self.param['feature_size'], dim, precision)
        for param_s in self.sampler.parameters():
            param_s.requires_grad = False
        self.register_buffer("queue_second", nn.functional.normalize(torch.randn(dim, K), dim=0))
        self.register_buffer("queue_vname", torch.ones(K, dtype=torch.long) * -1)
        self.register_buffer("queue_label", torch.ones(K, dtype=torch.long) * -1)
        self.queue_is_full = False
        self.reverse = reverse

    overlap_branches = True   # query, key and sampler encoders on three streams (they only share read-only inputs)

    def _qkf(self, x1, x2, f2):
        """The three encoder passes of a step -- query (gradient), key (shuffle-BN, no gradient) and the frozen sampler on
        the second view -- on three streams; they only share read-only inputs (reference pretrain.py:358-374 runs them
        one after the other)."""
        if not x1.is_cuda:
            raise moco.L.CoclrError("coclr_b200 modules run on CUDA (sm_90a) only; there is no CPU path")
        in_train_mode = torch.is_grad_enabled() and any(p.requires_grad for p in self.encoder_q.parameters())
        main = torch.cuda.current_stream()
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(priority=-1)     # key branch first: it carries the cross-rank exchange
        if getattr(self, "_side_stream2", None) is None:
            self._side_stream2 = torch.cuda.Stream()
        side = self._side_stream if CoCLR.overlap_branches else main
        side2 = self._side_stream2 if CoCLR.overlap_branches else main
        side.wait_stream(main)
        side2.wait_stream(main)
        overlap = side is not main
        if overlap:
            q = self.encoder_q.encode(x1)           # enqueued first (the key branch has host-side work, see InfoNCE._qk)
        with torch.cuda.stream(side), torch.no_grad():
            if in_train_mode:
                self._momentum_update_key_encoder()
            k, k_global = self._shuffled_keys(x2)
        with torch.cuda.stream(side2), torch.no_grad():
            kf = self.sampler.encode(f2)                                              # :372-374 (no shuffle)
        if not overlap:
            q = self.encoder_q.encode(x1)
        main.wait_stream(side)
        main.wait_stream(side2)
        for t in (k, k_global, kf):
            t.record_stream(main)
        return q, k, k_global, kf, in_train_mode

    def forward(self, block1, block2, k_vsource):
        x1, f1 = self._views(block1)
        x2, f2 = self._views(block2)
        if self.reverse:                                                              # :353-355
            x1, f1 = f1, x1
            x2, f2 = f2, x2
        q, k, k_global, kf, in_train_mode = self._qkf(x1, x2, f2)
        logits = moco.nce_logits(q, k, self.queue, self.T)
        if not self.queue_is_full:
            self.queue_is_full = bool(torch.all(self.queue_label != -1))              # :400-402
            if self.queue_is_full:
                print('\n===== queue is full now =====')
        # same-source positives OR the top-k of the second view's similarity (:392-413), one fused kernel
        mask = moco.mask_topk(kf, self.queue_second, k_vsource, self.queue_vname,
                              self.topk if self.queue_is_full else 0)
        if in_train_mode:
            with torch.no_grad():
                kf_global = concat_all_gather(kf)
                vn_global = concat_all_gather(k_vsource)
                ptr = self._dequeue_and_enqueue(k_global)
                n = k_global.shape[0]
                moco.enqueue(self.queue_second, kf_global.contiguous(), ptr)          # :334
                self.queue_vname[ptr:ptr + n] = vn_global                             # :335
                self.queue_label[ptr:ptr + n] = torch.ones_like(vn_global)            # :336
        return logits, mask
