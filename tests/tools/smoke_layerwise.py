"""Diagnostic (test infrastructure): the smoke() configuration (S3D, K=128, batch 2, 8 frames, 64x64) with every
post-BN activation of encoder_q / encoder_k compared against the float64 oracle and the float32 oracle.
  python tests/tools/smoke_layerwise.py [B] [T] [HW]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from model.pretrain import InfoNCE  # noqa: E402
from oracle import coclr_oracle as O  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 2
T = int(sys.argv[2]) if len(sys.argv) > 2 else 8
HW = int(sys.argv[3]) if len(sys.argv) > 3 else 64
K = 128
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
model = InfoNCE("s3d", 128, K)
sd = O.synth_state(O.infonce_shapes(128, K), seed=0, ptr=0)
model.load_state_dict(O.with_aliases(sd))
model = model.cuda().train()
g = torch.Generator().manual_seed(5)
block = torch.randn(B, 2, 3, T, HW, HW, generator=g).cuda()
torch.manual_seed(3)
idx = torch.randperm(B)
torch.manual_seed(3)
logits, labels = model(block)
torch.cuda.synchronize()


def oracle(dtype):
    rec = {}
    sdd = {k: (v.cuda().to(dtype) if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
    for k in O.param_keys(sdd, "encoder_q."):
        sdd[k].requires_grad_(True)
    orig = O._bn_relu

    def hook(s, pre, x, training):
        y = orig(s, pre, x, training)
        rec[pre] = y.detach()
        return y
    O._bn_relu = hook
    try:
        lg, _ = O.infonce_forward(sdd, [block.to(dtype)], idx)
    finally:
        O._bn_relu = orig
    return lg[0].detach(), rec


lg64, rec64 = oracle(torch.float64)
lg32, rec32 = oracle(torch.float32)
rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))
mx = lambda a, b: float((a.double() - b.double()).abs().max() / b.double().abs().max())
print("logits: ours %.3e  fp32 oracle %.3e (max-rel vs fp64)" % (mx(logits, lg64), mx(lg32, lg64)))
for enc, mod in (("encoder_q.", model.encoder_q), ("encoder_k.", model.encoder_k)):
    eng = mod._engine
    plan = [p for k, p in eng.plans.items() if k[0] == B][0]
    for t in eng.graph.tensors:
        if not t.pending:
            continue
        y = plan.acts[t.index].pl.value()
        for nm, coff, c in t.bn_members:
            key = enc + nm
            if key not in rec64:
                continue
            ref = rec64[key].permute(0, 2, 3, 4, 1)
            e = rel(y[..., coff:coff + c], ref)
            e32 = rel(rec32[key].permute(0, 2, 3, 4, 1), ref)
            flag = "  <<<" if e > 20 * max(e32, 1e-7) else ""
            print("%-46s %-18s ours %.2e  fp32 %.2e%s" % (key, tuple(ref.shape[1:4]), e, e32, flag))
    if enc == "encoder_k.":
        break
