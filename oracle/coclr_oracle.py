"""CPU/torch restatement of the CoCLR hot path -- TEST INFRASTRUCTURE ONLY.

This file is the parity oracle: a functional (state-dict driven) restatement of the reference's
S3D encoder + MoCo/InfoNCE step in stock PyTorch ops.  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import it; the product (coclr_b200/, model/,
backbone/) never does.

Pinned against what the UNMODIFIED reference modules computed (bit-for-bit on logits / loss / queue / masks, to 1e-6 on
the recorded post-step state):
  tests/test_oracle.py       InfoNCE with the S3D and the ResNet2d3d-50 backbone; adam_step against torch.optim.Adam
  tests/test_oracle_ext.py   UberNCE, CoCLR (queue warm-up and queue-full phases, top-k mining)
  tests/test_oracle_dist.py  the simulated multi-rank world against the reference run as two gloo DDP ranks
tests/golden/*.npz hold the reference outputs produced by tests/golden/make_golden*.py (run with COCLR_REFERENCE
pointing at a reference checkout); the tests check the oracle against them.

Every function cites the reference file:line it restates (paths relative to TengdaHan/CoCLR).
State is a flat dict {state_dict key: tensor} with exactly the reference's key names, e.g.
'encoder_q.0.Conv_1a.conv1.weight', 'encoder_q.2.bias', 'queue', 'queue_ptr'.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5        # nn.BatchNorm3d default, backbone/s3dg.py:16,46-47
BN_MOMENTUM = 0.1

# SepInception output planes [b0, b1a, b1b, b2a, b2b, b3b]; backbone/s3dg.py:163-164,174-178,191-192
INCEPTION = [
    ("Mixed_3b", 192, [64, 96, 128, 16, 32, 32]),
    ("Mixed_3c", 256, [128, 128, 192, 32, 96, 64]),
    ("Mixed_4b", 480, [192, 96, 208, 16, 48, 64]),
    ("Mixed_4c", 512, [160, 112, 224, 24, 64, 64]),
    ("Mixed_4d", 512, [128, 128, 256, 24, 64, 64]),
    ("Mixed_4e", 512, [112, 144, 288, 32, 64, 64]),
    ("Mixed_4f", 528, [256, 160, 320, 32, 128, 128]),
    ("Mixed_5b", 832, [256, 160, 320, 32, 128, 128]),
    ("Mixed_5c", 832, [384, 192, 384, 48, 128, 128]),
]


def _bn_relu(sd, pre, x, training):
    """nn.BatchNorm3d (train: batch stats + running update; eval: running stats) then ReLU;
    backbone/s3dg.py:16-17,24-27."""
    rm, rv = sd[pre + ".running_mean"], sd[pre + ".running_var"]
    if training:
        sd[pre + ".num_batches_tracked"] += 1
    y = F.batch_norm(x, rm, rv, sd[pre + ".weight"], sd[pre + ".bias"], training, BN_MOMENTUM, BN_EPS)
    return F.relu(y)


def basic_conv(sd, pre, x, training):
    """BasicConv3d: 1x1x1 conv (no bias) -> BN -> ReLU; backbone/s3dg.py:8-28."""
    x = F.conv3d(x, sd[pre + ".conv.weight"])
    return _bn_relu(sd, pre + ".bn", x, training)


def st_conv(sd, pre, x, k, stride, t_stride, pad, training):
    """STConv3d: (1,k,k) conv -> BN -> ReLU -> (k,1,1) conv -> BN -> ReLU; backbone/s3dg.py:30-65."""
    x = F.conv3d(x, sd[pre + ".conv1.weight"], stride=(1, stride, stride), padding=(0, pad, pad))
    x = _bn_relu(sd, pre + ".bn1", x, training)
    x = F.conv3d(x, sd[pre + ".conv2.weight"], stride=(t_stride, 1, 1), padding=(pad, 0, 0))
    return _bn_relu(sd, pre + ".bn2", x, training)


def self_gating(sd, pre, x):
    """SelfGating ("feature gating as used in S3D-G"): sigmoid(fc(mean over T,H,W)) scales every channel of every clip;
    backbone/s3dg.py:68-78."""
    avg = torch.mean(x, dim=[2, 3, 4])                                              # :75
    w = torch.sigmoid(F.linear(avg, sd[pre + ".fc.weight"], sd[pre + ".fc.bias"]))  # :76-77
    return w[:, :, None, None, None] * x                                            # :78


def sep_inception(sd, pre, x, training):
    """SepInception: 4 branches concatenated on channels; backbone/s3dg.py:81-132.  With gating (network 's3dg',
    select_backbone.py:8-9; recognised from the state keys) each branch output goes through its SelfGating (:125-129)."""
    x0 = basic_conv(sd, pre + ".branch0.0", x, training)
    x1 = basic_conv(sd, pre + ".branch1.0", x, training)
    x1 = st_conv(sd, pre + ".branch1.1", x1, 3, 1, 1, 1, training)
    x2 = basic_conv(sd, pre + ".branch2.0", x, training)
    x2 = st_conv(sd, pre + ".branch2.1", x2, 3, 1, 1, 1, training)
    x3 = F.max_pool3d(x, kernel_size=(3, 3, 3), stride=1, padding=1)
    x3 = basic_conv(sd, pre + ".branch3.1", x3, training)
    if (pre + ".gating_b0.fc.weight") in sd:                                        # :124
        x0 = self_gating(sd, pre + ".gating_b0", x0)
        x1 = self_gating(sd, pre + ".gating_b1", x1)
        x2 = self_gating(sd, pre + ".gating_b2", x2)
        x3 = self_gating(sd, pre + ".gating_b3", x3)
    return torch.cat((x0, x1, x2, x3), 1)


def s3d(sd, pre, x, training):
    """S3D.forward; backbone/s3dg.py:135-217 (block1..block5)."""
    x = st_conv(sd, pre + "Conv_1a", x, 7, 2, 2, 3, training)                       # :145
    x = F.max_pool3d(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))                            # :151
    x = basic_conv(sd, pre + "Conv_2b", x, training)                                # :152
    x = st_conv(sd, pre + "Conv_2c", x, 3, 1, 1, 1, training)                       # :153
    x = F.max_pool3d(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))                            # :162
    for name, _, _ in INCEPTION[:2]:
        x = sep_inception(sd, pre + name, x, training)
    x = F.max_pool3d(x, (3, 3, 3), (2, 2, 2), (1, 1, 1))                            # :173
    for name, _, _ in INCEPTION[2:7]:
        x = sep_inception(sd, pre + name, x, training)
    x = F.max_pool3d(x, (2, 2, 2), (2, 2, 2), (0, 0, 0))                            # :190
    for name, _, _ in INCEPTION[7:]:
        x = sep_inception(sd, pre + name, x, training)
    return x


# ---------------------------------------------------------------------------------------------
# ResNet2d3d-50 ("r50", BASELINE.json config 5); backbone/resnet_2d3d.py
# ---------------------------------------------------------------------------------------------
R50_LAYERS = [("layer1", 64, 3, 1, False), ("layer2", 128, 4, 2, False),      # (name, planes, blocks, stride, 3d?)
              ("layer3", 256, 6, 2, True), ("layer4", 512, 3, 2, True)]        # resnet_2d3d.py:143-146,204-208


def _bn(sd, pre, x, training):
    """nn.BatchNorm3d without the ReLU (bn3 / downsample BN of a bottleneck)."""
    if training:
        sd[pre + ".num_batches_tracked"] += 1
    return F.batch_norm(x, sd[pre + ".running_mean"], sd[pre + ".running_var"], sd[pre + ".weight"], sd[pre + ".bias"],
                        training, BN_MOMENTUM, BN_EPS)


def bottleneck(sd, pre, x, stride, is3d, training):
    """Bottleneck2d (conv1 1x1x1) / Bottleneck3d (conv1 (3,1,1), pad (1,0,0)) -> (1,3,3) conv with the spatial
    stride -> 1x1x1 conv x4, residual add (through the 1x1x1 strided downsample conv + BN when present), ReLU;
    backbone/resnet_2d3d.py:46-131.  The last block of layer4 skips its own ReLU (:183-185) but ResNet2d3d.forward
    ends with F.relu (:202), so every block is followed by exactly one ReLU."""
    out = F.conv3d(x, sd[pre + ".conv1.weight"], padding=(1, 0, 0) if is3d else 0)
    out = F.relu(_bn(sd, pre + ".bn1", out, training))
    out = F.conv3d(out, sd[pre + ".conv2.weight"], stride=(1, stride, stride), padding=(0, 1, 1))
    out = F.relu(_bn(sd, pre + ".bn2", out, training))
    out = _bn(sd, pre + ".bn3", F.conv3d(out, sd[pre + ".conv3.weight"]), training)
    if (pre + ".downsample.0.weight") in sd:
        x = F.conv3d(x, sd[pre + ".downsample.0.weight"], stride=(1, stride, stride))
        x = _bn(sd, pre + ".downsample.1", x, training)
    return F.relu(out + x)


def r2d3d50(sd, pre, x, training):
    """ResNet2d3d([Bottleneck2d, Bottleneck2d, Bottleneck3d, Bottleneck3d], [3, 4, 6, 3]).forward;
    backbone/resnet_2d3d.py:133-202."""
    x = F.conv3d(x, sd[pre + "conv1.weight"], stride=(2, 2, 2), padding=(2, 3, 3))      # :138
    x = F.relu(_bn(sd, pre + "bn1", x, training))
    x = F.max_pool3d(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))                                # :141
    for name, _, blocks, stride, is3d in R50_LAYERS:
        for i in range(blocks):
            x = bottleneck(sd, "%s%s.%d" % (pre, name, i), x, stride if i == 0 else 1, is3d, training)
    return x


def r50_shapes(pre, first_channel=3):
    """{key: shape} of an r2d3d50 backbone under prefix `pre` (parameters and BN buffers)."""
    sh = {}

    def bn(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)
        sh[p + ".running_mean"] = (c,)
        sh[p + ".running_var"] = (c,)
        sh[p + ".num_batches_tracked"] = ()

    sh[pre + "conv1.weight"] = (64, first_channel, 5, 7, 7)
    bn(pre + "bn1", 64)
    inplanes = 64
    for name, planes, blocks, stride, is3d in R50_LAYERS:
        for i in range(blocks):
            p = "%s%s.%d" % (pre, name, i)
            sh[p + ".conv1.weight"] = (planes, inplanes, 3 if is3d else 1, 1, 1)
            bn(p + ".bn1", planes)
            sh[p + ".conv2.weight"] = (planes, planes, 1, 3, 3)
            bn(p + ".bn2", planes)
            sh[p + ".conv3.weight"] = (planes * 4, planes, 1, 1, 1)
            bn(p + ".bn3", planes * 4)
            if i == 0:                                                                   # :151-165
                sh[p + ".downsample.0.weight"] = (planes * 4, inplanes, 1, 1, 1)
                bn(p + ".downsample.1", planes * 4)
            inplanes = planes * 4
    return sh



def encoder(sd, pre, x, training):
    """backbone -> AdaptiveAvgPool3d(1) -> Conv3d(fs,fs,1,bias) -> ReLU -> Conv3d(fs,dim,1,bias), fs = 1024 (s3d) /
    2048 (r50); model/pretrain.py:49-54. Returns [B, dim, 1, 1, 1]. The backbone is recognised from the state keys."""
    backbone = r2d3d50 if (pre + "0.layer1.0.conv1.weight") in sd else s3d       # select_backbone.py:4-16
    f = backbone(sd, pre + "0.", x, training)
    f = F.adaptive_avg_pool3d(f, (1, 1, 1))
    f = F.relu(F.conv3d(f, sd[pre + "2.weight"], sd[pre + "2.bias"]))
    return F.conv3d(f, sd[pre + "4.weight"], sd[pre + "4.bias"])


def param_keys(sd, pre):
    """Keys that nn.Module.parameters() would yield for an encoder (weights/biases, no BN buffers)."""
    return [k for k in sd if k.startswith(pre) and (k.endswith(".weight") or k.endswith(".bias"))]


@torch.no_grad()
def momentum_update(sd, m):
    """_momentum_update_key_encoder: k = k*m + q*(1-m) over parameters only; model/pretrain.py:76-80."""
    for kq in param_keys(sd, "encoder_q."):
        kk = "encoder_k." + kq[len("encoder_q."):]
        sd[kk] = sd[kk] * m + sd[kq].detach() * (1. - m)


def infonce_forward(sd, blocks, idx_shuffle, m=0.999, T=0.07, training=True, keep_graph=True):
    """InfoNCE.forward for a simulated world of len(blocks) ranks sharing `sd`; model/pretrain.py:145-190.

    blocks: list (one per rank) of [B,2,C,T,H,W]; idx_shuffle: the permutation rank 0 would broadcast
    (pretrain.py:112-115).  Returns (list of logits per rank, labels).  Side effects on sd as in the
    reference: EMA of encoder_k (:161), BN running statistics, queue / queue_ptr (:82-96).
    BN buffers tracked are rank 0's (DDP re-broadcasts rank 0's buffers before every forward).
    keep_graph=False (checker use only, e.g. bench.py's parity block over 8 simulated ranks): the query features are
    detached as soon as they are computed, so that only one encoder pass of activations is alive at a time; every
    value and side effect is the same, only backward through the returned logits is unavailable.
    """
    W = len(blocks)
    B = blocks[0].shape[0]
    dim = sd["queue"].shape[0]
    for blk in blocks:
        assert blk.shape[1] == 2                                                    # :148
    # queries (:153-155); BN buffer side effects kept for rank 0 only
    qs = []
    in_train_mode = None
    for r, blk in enumerate(blocks):
        sdr = sd if r == 0 else _bn_scratch(sd, "encoder_q.")
        q = encoder(sdr, "encoder_q.", blk[:, 0].contiguous(), training)
        q = F.normalize(q, dim=1).view(B, dim)
        if in_train_mode is None:
            in_train_mode = q.requires_grad                                         # :157
        qs.append(q if keep_graph else q.detach())
    with torch.no_grad():
        if in_train_mode:
            momentum_update(sd, m)                                                  # :161
        x_all = torch.cat([blk[:, 1] for blk in blocks], 0)                         # :105-106
        idx_unshuffle = torch.argsort(idx_shuffle)                                  # :118
        k_sh = []
        for r in range(W):
            idx_this = idx_shuffle.view(W, -1)[r]                                   # :121-124
            sdr = sd if r == 0 else _bn_scratch(sd, "encoder_k.")
            k = encoder(sdr, "encoder_k.", x_all[idx_this].contiguous(), True if training else False)
            k_sh.append(F.normalize(k, dim=1))
        k_all = torch.cat(k_sh, 0)[idx_unshuffle].view(W * B, dim)                  # :133-143
    queue0 = sd["queue"].clone().detach()
    logits = []
    for r in range(W):
        k = k_all[r * B:(r + 1) * B]
        l_pos = torch.einsum('nc,nc->n', [qs[r], k]).unsqueeze(-1)                  # :175
        l_neg = torch.einsum('nc,ck->nk', [qs[r], queue0])                          # :176
        lg = torch.cat([l_pos, l_neg], dim=1)                                       # :179
        logits.append(lg / T)                                                       # :182
    labels = torch.zeros(B, dtype=torch.long)                                       # :185
    if in_train_mode:
        with torch.no_grad():                                                       # :82-96
            ptr = int(sd["queue_ptr"])
            K = sd["queue"].shape[1]
            assert K % (W * B) == 0
            sd["queue"][:, ptr:ptr + W * B] = k_all.T
            sd["queue_ptr"][0] = (ptr + W * B) % K
    return logits, labels


def _bn_scratch(sd, pre):
    """View of sd in which the BN buffers under `pre` are private copies (non-zero ranks)."""
    out = dict(sd)
    for k, v in sd.items():
        if k.startswith(pre) and (k.endswith("running_mean") or k.endswith("running_var")
                                  or k.endswith("num_batches_tracked")):
            out[k] = v.clone()
    return out


def infonce_loss(logits, labels):
    """nn.CrossEntropyLoss() on (logits, labels); main_nce.py:201,314."""
    return F.cross_entropy(logits, labels)


def adam_step(params, grads, state, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5):
    """torch.optim.Adam with coupled L2 weight decay on every tensor; main_nce.py:190-200.
    state: dict key -> {'step', 'exp_avg', 'exp_avg_sq'} (created on first use)."""
    b1, b2 = betas
    with torch.no_grad():
        for k in params:
            g = grads[k]
            if g is None:
                continue
            p = params[k]
            st = state.setdefault(k, {"step": 0, "exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)})
            st["step"] += 1
            g = g.add(p, alpha=weight_decay)
            st["exp_avg"].lerp_(g, 1 - b1)
            st["exp_avg_sq"].mul_(b2).addcmul_(g, g.conj(), value=1 - b2)
            bc1 = 1 - b1 ** st["step"]
            bc2 = 1 - b2 ** st["step"]
            denom = (st["exp_avg_sq"].sqrt() / (bc2 ** 0.5)).add_(eps)
            p.addcdiv_(st["exp_avg"], denom, value=-(lr / bc1))


# ---------------------------------------------------------------------------------------------
# shapes + deterministic synthetic state (shared by the golden generator and the tests)
# ---------------------------------------------------------------------------------------------
def s3d_shapes(pre, first_channel=3, gating=False):
    """{key: shape} of an S3D backbone under prefix `pre` (parameters and BN buffers); gating: the S3D-G variant."""
    sh = {}

    def bn(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)
        sh[p + ".running_mean"] = (c,)
        sh[p + ".running_var"] = (c,)
        sh[p + ".num_batches_tracked"] = ()

    def basic(p, ci, co):
        sh[p + ".conv.weight"] = (co, ci, 1, 1, 1)
        bn(p + ".bn", co)

    def st(p, ci, co, k):
        sh[p + ".conv1.weight"] = (co, ci, 1, k, k)
        sh[p + ".conv2.weight"] = (co, co, k, 1, 1)
        bn(p + ".bn1", co)
        bn(p + ".bn2", co)

    st(pre + "Conv_1a", first_channel, 64, 7)
    basic(pre + "Conv_2b", 64, 64)
    st(pre + "Conv_2c", 64, 192, 3)
    for name, cin, (o0, o1a, o1b, o2a, o2b, o3b) in INCEPTION:
        basic(pre + name + ".branch0.0", cin, o0)
        basic(pre + name + ".branch1.0", cin, o1a)
        st(pre + name + ".branch1.1", o1a, o1b, 3)
        basic(pre + name + ".branch2.0", cin, o2a)
        st(pre + name + ".branch2.1", o2a, o2b, 3)
        basic(pre + name + ".branch3.1", cin, o3b)
        if gating:                                                                   # s3dg.py:107-112
            for i, c in enumerate((o0, o1b, o2b, o3b)):
                sh["%s%s.gating_b%d.fc.weight" % (pre, name, i)] = (c, c)
                sh["%s%s.gating_b%d.fc.bias" % (pre, name, i)] = (c,)
    return sh


def infonce_shapes(dim=128, K=2048, feature_size=None, network="s3d"):
    sh = {}
    feature_size = feature_size or {"s3d": 1024, "s3dg": 1024, "r50": 2048}[network]
    for enc in ("encoder_q.", "encoder_k."):
        sh.update(r50_shapes(enc + "0.") if network == "r50" else s3d_shapes(enc + "0.", gating=network == "s3dg"))
        sh[enc + "2.weight"] = (feature_size, feature_size, 1, 1, 1)
        sh[enc + "2.bias"] = (feature_size,)
        sh[enc + "4.weight"] = (dim, feature_size, 1, 1, 1)
        sh[enc + "4.bias"] = (dim,)
    sh["queue"] = (dim, K)
    sh["queue_ptr"] = (1,)
    return sh


def synth_state(shapes, seed=0, ptr=0, k_delta=0.02):
    """Deterministic 'warmed-up' state: He-like conv weights, non-trivial BN affine/buffers,
    encoder_k = encoder_q + small perturbation, unit-norm queue columns."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k in sorted(shapes):
        s = tuple(shapes[k])
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(3, dtype=torch.long)
        elif k == "queue_ptr":
            sd[k] = torch.tensor([ptr], dtype=torch.long)
        elif k == "queue":
            sd[k] = F.normalize(torch.randn(s, generator=g), dim=0)
        elif k.endswith("running_var"):
            sd[k] = torch.rand(s, generator=g) + 0.5
        elif k.endswith("running_mean"):
            sd[k] = torch.randn(s, generator=g) * 0.1
        elif (".bn" in k or ".downsample.1." in k) and k.endswith(".weight"):
            sd[k] = torch.rand(s, generator=g) + 0.5
        elif ".bn" in k and k.endswith(".bias"):
            sd[k] = torch.randn(s, generator=g) * 0.1
        elif k.endswith(".bias"):
            sd[k] = torch.randn(s, generator=g) * 0.05
        elif len(s) == 2:  # nn.Linear weight of a SelfGating: gates spread over (0.2, 0.8) instead of all ~0.5
            sd[k] = torch.randn(s, generator=g) * (4.0 / s[1]) ** 0.5
        else:  # conv weight
            fan_in = s[1] * s[2] * s[3] * s[4]
            sd[k] = torch.randn(s, generator=g) * (2.0 / fan_in) ** 0.5
    for k in list(sd):
        if k.startswith("encoder_k.") and (k.endswith(".weight") or k.endswith(".bias")):
            q = sd["encoder_q." + k[len("encoder_k."):]]
            sd[k] = q + k_delta * q.abs().mean() * torch.randn(q.shape, generator=g)
    return sd


# The reference registers every backbone stage twice (self.Conv_1a and self.block1[0], ...;
# backbone/s3dg.py:145-192), so its state_dict carries alias keys 'blockN.i.*' for the same tensors.
BLOCK_ALIASES = {
    "Conv_1a": "block1.0", "Conv_2b": "block2.1", "Conv_2c": "block2.2",
    "Mixed_3b": "block3.1", "Mixed_3c": "block3.2",
    "Mixed_4b": "block4.1", "Mixed_4c": "block4.2", "Mixed_4d": "block4.3", "Mixed_4e": "block4.4",
    "Mixed_4f": "block4.5", "Mixed_5b": "block5.1", "Mixed_5c": "block5.2",
}


def with_aliases(sd):
    """Return sd plus the reference's 'blockN.i' alias keys (same tensor objects)."""
    out = dict(sd)
    for k, v in sd.items():
        parts = k.split(".")
        for i, p in enumerate(parts):
            if p in BLOCK_ALIASES and i >= 1 and parts[i - 1] == "0":
                out[".".join(parts[:i] + [BLOCK_ALIASES[p]] + parts[i + 1:])] = v
                break
    return out


# ---------------------------------------------------------------------------------------------
# UberNCE and CoCLR (single simulated rank; the shuffle algebra is covered by infonce_forward)
# ---------------------------------------------------------------------------------------------
def _qk_single(sd, x1, x2, idx_shuffle, m, training):
    """Shared q / k computation of the three models at world size 1 (model/pretrain.py:153-170,246-262,357-370)."""
    B = x1.shape[0]
    dim = sd["queue"].shape[0]
    q = F.normalize(encoder(sd, "encoder_q.", x1.contiguous(), training), dim=1).view(B, dim)
    in_train_mode = q.requires_grad
    with torch.no_grad():
        if in_train_mode:
            momentum_update(sd, m)
        idx_unshuffle = torch.argsort(idx_shuffle)
        k = F.normalize(encoder(sd, "encoder_k.", x2[idx_shuffle].contiguous(), training), dim=1)
        k = k[idx_unshuffle].view(B, dim)
    return q, k, in_train_mode


def _logits(sd, q, k, T):
    l_pos = torch.einsum('nc,nc->n', [q, k]).unsqueeze(-1)
    l_neg = torch.einsum('nc,ck->nk', [q, sd["queue"].clone().detach()])
    return torch.cat([l_pos, l_neg], dim=1) / T


def ubernce_forward(sd, block, k_label, idx_shuffle, m=0.999, T=0.07, training=True):
    """UberNCE.forward (model/pretrain.py:230-278) + its _dequeue_and_enqueue (:211-227). Returns (logits, mask)."""
    assert block.shape[1] == 2
    q, k, in_train_mode = _qk_single(sd, block[:, 0], block[:, 1], idx_shuffle, m, training)
    logits = _logits(sd, q, k, T)
    mask = k_label.unsqueeze(1) == sd["queue_label"].unsqueeze(0)                                # :271
    mask = torch.cat([torch.ones((mask.shape[0], 1), dtype=torch.bool), mask], dim=1)            # :272-273
    if in_train_mode:
        with torch.no_grad():
            ptr = int(sd["queue_ptr"])
            B, K = k.shape[0], sd["queue"].shape[1]
            assert K % B == 0
            sd["queue"][:, ptr:ptr + B] = k.T
            sd["queue_label"][ptr:ptr + B] = k_label                                             # :224
            sd["queue_ptr"][0] = (ptr + B) % K
    return logits, mask


def coclr_forward(sd, block1, block2, k_vsource, idx_shuffle, queue_is_full, topk=5, reverse=False, m=0.999, T=0.07,
                  training=True, sampler_training=False):
    """CoCLR.forward (model/pretrain.py:344-418) + _dequeue_and_enqueue (:321-341).
    Returns (logits, mask, queue_is_full). The sampler runs with eval-mode BN (main_coclr.py:363)."""
    B = block1.shape[0]
    dim = sd["queue"].shape[0]
    x1, f1 = block1[:, 0], block1[:, 1]                                                          # :347-350
    x2, f2 = block2[:, 0], block2[:, 1]
    if reverse:                                                                                  # :353-355
        x1, f1 = f1, x1
        x2, f2 = f2, x2
    q, k, in_train_mode = _qk_single(sd, x1, x2, idx_shuffle, m, training)
    with torch.no_grad():
        kf = F.normalize(encoder(sd, "sampler.", f2.contiguous(), sampler_training), dim=1).view(B, dim)   # :372-374
    logits = _logits(sd, q, k, T)
    mask_source = k_vsource.unsqueeze(1) == sd["queue_vname"].unsqueeze(0)                       # :392
    mask = mask_source.clone()
    if not queue_is_full:                                                                        # :400-402
        queue_is_full = bool(torch.all(sd["queue_label"] != -1))
    if queue_is_full and topk != 0:                                                              # :404-410
        mask_sim = kf.matmul(sd["queue_second"].clone().detach())
        mask_sim[mask_source] = -float("inf")
        _, topkidx = torch.topk(mask_sim, topk, dim=1)
        topk_onehot = torch.zeros_like(mask_sim)
        topk_onehot.scatter_(1, topkidx, 1)
        mask[topk_onehot.bool()] = True
    mask = torch.cat([torch.ones((mask.shape[0], 1), dtype=torch.bool), mask], dim=1)
    if in_train_mode:
        with torch.no_grad():                                                                    # :321-341
            ptr = int(sd["queue_ptr"])
            K = sd["queue"].shape[1]
            assert K % B == 0
            sd["queue"][:, ptr:ptr + B] = k.T
            sd["queue_second"][:, ptr:ptr + B] = kf.T
            sd["queue_vname"][ptr:ptr + B] = k_vsource
            sd["queue_label"][ptr:ptr + B] = torch.ones_like(k_vsource)
            sd["queue_ptr"][0] = (ptr + B) % K
    return logits, mask.detach(), queue_is_full


def coclr_shapes(dim=128, K=2048, feature_size=None, network="s3d"):
    sh = infonce_shapes(dim, K, feature_size, network)
    sh.update({"sampler." + k[len("encoder_q."):]: v for k, v in sh.items() if k.startswith("encoder_q.")})
    sh["queue_second"] = (dim, K)
    sh["queue_vname"] = (K,)
    sh["queue_label"] = (K,)
    return sh


def synth_state_ext(shapes, seed=0, ptr=0, full=True, n_ids=12):
    """synth_state plus the integer queues of UberNCE / CoCLR: labels / video ids drawn from a small range so that
    positives exist; `full` decides whether queue_label still contains -1 (CoCLR's warm-up phase)."""
    base = {k: v for k, v in shapes.items() if k not in ("queue_second", "queue_vname", "queue_label")}
    sd = synth_state(base, seed=seed, ptr=ptr)
    g = torch.Generator().manual_seed(seed + 17)
    K = shapes["queue"][1]
    if "queue_second" in shapes:
        sd["queue_second"] = F.normalize(torch.randn(shapes["queue_second"], generator=g), dim=0)
    if "queue_vname" in shapes:
        sd["queue_vname"] = torch.randint(0, n_ids, (K,), generator=g)
    if "queue_label" in shapes:
        lab = torch.randint(0, n_ids, (K,), generator=g)
        if not full:
            lab[K // 2:] = -1
        sd["queue_label"] = lab
    for k in list(sd):
        if k.startswith("sampler.") and (k.endswith(".weight") or k.endswith(".bias")):
            sd[k] = sd[k] + 0.05 * sd[k].abs().mean() * torch.randn(sd[k].shape, generator=g)
    return sd
