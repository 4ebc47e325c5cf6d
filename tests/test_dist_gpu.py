"""2-GPU (NCCL) parity of the data-parallel InfoNCE step against the oracle's simulated 2-rank world
(oracle.infonce_forward with two blocks; model/pretrain.py:98-143 shuffle-BN, :82-96 enqueue; DDP gradient averaging
main_nce.py:172): per-rank logits, the replicated queue, and replica-identical weights after the all-reduced Adam step.
Needs two visible GPUs (skipped on the 1-GPU round-end box; run with `gpurun --gpus 2`)."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

B, T, HW, K, PTR = 4, 8, 128, 128, 16


def _blocks():
    out = []
    for r in range(2):
        g = torch.Generator().manual_seed(4321 + r)
        out.append(torch.randn(B, 2, 3, T, HW, HW, generator=g))
    return out


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from model.pretrain import InfoNCE
    from coclr_b200 import moco
    from oracle import coclr_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = O.synth_state(O.infonce_shapes(128, K), seed=0, ptr=PTR)
    model = InfoNCE("s3d", 128, K, 0.999, 0.07)
    model.load_state_dict(O.with_aliases(sd), strict=True)
    model = model.to(dev).train()
    opt = moco.FlatAdam(model.encoder_q, lr=1e-3, weight_decay=1e-5)
    blocks = _blocks()
    torch.manual_seed(77 + 1000 * rank)      # ranks draw different permutations; rank 0's is broadcast (pretrain.py:112-115)
    logits, labels = model(blocks[rank].to(dev))
    loss = moco.nce_cross_entropy(logits, labels)
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    # ---- oracle: the same 2-rank world simulated on this GPU in float64 ----
    torch.manual_seed(77)
    idx = torch.randperm(B * world)
    sdd = {k: (v.detach().clone().to(dev).double() if v.is_floating_point() else v.clone().to(dev)) for k, v in sd.items()}
    qkeys = O.param_keys(sdd, "encoder_q.")
    for k in qkeys:
        sdd[k].requires_grad_(True)
    lgs, lab = O.infonce_forward(sdd, [b.to(dev).double() for b in blocks], idx.to(dev))
    losses = [O.infonce_loss(lg, lab.to(dev)) for lg in lgs]
    (sum(losses) / world).backward()                  # DDP averages the per-rank gradients
    rel = lambda a, b: float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))
    res = {"logits_err": rel(logits, lgs[rank]), "queue_err": rel(model.queue, sdd["queue"]),
           "ptr": int(model.queue_ptr), "ptr_ref": int(sdd["queue_ptr"]),
           "loss": float(loss), "loss_ref": float(losses[rank])}
    # all-reduced gradient (sum over ranks, 1/W folded into Adam) vs the oracle's averaged gradient, per tensor
    st = model.encoder_q._engine.store
    errs = []
    for k in qkeys:
        name = k[len("encoder_q."):]
        g_new = st.view(name, grad=True) / world
        errs.append(float((g_new.double() - sdd[k].grad).norm() / sdd[k].grad.norm().clamp_min(1e-30)))
    errs.sort()
    res["grad_median"], res["grad_max"] = errs[len(errs) // 2], errs[-1]
    # replicas stay identical: compare flat parameters and Adam moments across ranks
    flat = st.flat.clone()
    other = flat.clone()
    dist.broadcast(other, src=0)
    res["replica_identical"] = bool(torch.equal(flat, other))
    qk = model.queue.clone()
    dist.broadcast(qk, src=0)
    res["queue_identical"] = bool(torch.equal(qk, model.queue))
    torch.save(res, os.path.join(out, "rank%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (gpurun --gpus 2)")
@pytest.mark.timeout(900)
def test_infonce_step_world2_nccl(tmp_path, diag):
    port = 29600 + (os.getpid() % 300)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r = [torch.load(os.path.join(str(tmp_path), "rank%d.pt" % i)) for i in range(2)]
    diag["dist2/results"] = r
    for x in r:
        assert x["logits_err"] < 1e-3, x
        assert x["queue_err"] < 1e-3 and x["ptr"] == x["ptr_ref"] == PTR + 2 * B
        assert abs(x["loss"] - x["loss_ref"]) < 1e-3 * max(1.0, abs(x["loss_ref"]))
        assert x["replica_identical"] and x["queue_identical"]
        assert x["grad_median"] < 0.15 and x["grad_max"] < 0.5, x
