"""Measurement tool (test infrastructure, not product): times the oracle -- the reference's algorithm in stock
PyTorch ops -- on the GPU, i.e. what the unmodified reference would do on this GPU through cuDNN/cuBLAS.
Reported next to our numbers as "the kernel to beat" (SURVEY.md 2a).  Usage:
    python tests/tools/bench_torch_gpu.py [--batch 32] [--steps 5] [--mode fp32|tf32|bf16]"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import coclr_oracle as O  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--seq_len", type=int, default=32)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--mode", default="tf32")
args = ap.parse_args()

tf32 = args.mode != "fp32"
torch.backends.cudnn.allow_tf32 = tf32
torch.backends.cuda.matmul.allow_tf32 = tf32
torch.backends.cudnn.benchmark = True
dev = torch.device("cuda")
K = 2048
sd = {k: v.to(dev) for k, v in O.synth_state(O.infonce_shapes(128, K), seed=0).items()}
qkeys = O.param_keys(sd, "encoder_q.")
for k in qkeys:
    sd[k].requires_grad_(True)
state = {}
block = torch.randn(args.batch, 2, 3, args.seq_len, 128, 128, device=dev)


def step():
    idx = torch.randperm(args.batch)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(args.mode == "bf16")):
        logits, labels = O.infonce_forward(sd, [block], idx.to(dev))
        loss = O.infonce_loss(logits[0].float(), labels.to(dev))
    grads = torch.autograd.grad(loss, [sd[k] for k in qkeys])
    O.adam_step({k: sd[k] for k in qkeys}, dict(zip(qkeys, grads)), state)


for _ in range(2):
    step()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(args.steps):
    step()
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / args.steps
print(json.dumps({"impl": "stock-pytorch-on-gpu (oracle ops via cuDNN/cuBLAS)", "mode": args.mode, "batch": args.batch,
                  "ms_per_step": dt * 1e3, "clips_per_s": 2 * args.batch / dt,
                  "torch": torch.__version__, "cudnn": torch.backends.cudnn.version()}))
