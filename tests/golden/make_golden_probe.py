"""Writes tests/golden/feature_probe.npz by running the UNMODIFIED reference eval/feature_linear_probe.py
($COCLR_REFERENCE) on the CPU over seeded small features.

The script is run as is: `.cuda()` of tensors and modules is patched to identity (the module patch also records the LP
it is called on, whose state_dict() after the run is the final model), and matplotlib, which the script imports but does
not use, is stubbed.  Three cases cover --final_bn on and off, --normalize, partial last batches (one of a single row,
without BN) and eval_freq > 1.  Per case the file holds the inputs, the flags, the initial and final state dicts, the printed lines
and the saved probability JSON (as [Nq, C] in vname order).

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_probe.py
"""
import contextlib
import io
import json
import os
import pickle
import runpy
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402

OUT = os.path.join(HERE, "feature_probe.npz")
# name -> (N, Nq, D, C, seed, flags)
CASES = {
    "bn": (150, 61, 32, 5, 11, ["--final_bn", "--batch_size", "32", "--epochs", "8", "--eval_freq", "3",
                                "--schedule", "4", "6", "--lr", "0.5", "--wd", "1e-3"]),
    "norm": (129, 60, 32, 5, 12, ["--normalize", "--batch_size", "32", "--epochs", "6", "--eval_freq", "2",
                                  "--schedule", "3", "5", "--lr", "1.0", "--wd", "1e-2"]),
    "bn_norm": (150, 61, 32, 5, 13, ["--final_bn", "--normalize", "--batch_size", "64", "--epochs", "5",
                                     "--eval_freq", "1", "--schedule", "3", "--lr", "0.3", "--wd", "1e-4"]),
}


def features(N, Nq, D, C, seed):
    """Overlapping classes (accuracies well below 1): class means of scale 0.35 under unit noise, with an offset and
    uneven column scales so that BatchNorm has something to do."""
    g = torch.Generator().manual_seed(seed)
    means = 0.35 * torch.randn(C, D, generator=g)
    scale = torch.rand(D, generator=g) * 2 + 0.5
    offset = torch.randn(D, generator=g)

    def split(n):
        y = torch.arange(n) % C
        y = y[torch.randperm(n, generator=g)]
        return (means[y] + torch.randn(n, D, generator=g)) * scale + offset, y

    xtr, ytr = split(N)
    xte, yte = split(Nq)
    return xtr, ytr, xte, yte


def run_reference(d, flags):
    script = os.path.join(REF, "eval", "feature_linear_probe.py")
    models = []
    saved = (torch.Tensor.cuda, nn.Module.cuda, sys.argv, list(sys.path), dict(sys.modules))

    def module_cuda(self, *a, **k):   # called on the LP right after it is built: record its initial state too
        models.append((self, {k: v.clone() for k, v in self.state_dict().items()}))
        return self

    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot.switch_backend = lambda *a, **k: None
    try:
        torch.Tensor.cuda = lambda self, *a, **k: self
        nn.Module.cuda = module_cuda
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
        sys.path.insert(0, REF)
        sys.argv = [script, "--test", os.path.join(d, "model.pth.tar")] + flags
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            runpy.run_path(script, run_name="__main__")
    finally:
        torch.Tensor.cuda, nn.Module.cuda, sys.argv = saved[0], saved[1], saved[2]
        sys.path[:] = saved[3]
        for k in list(sys.modules):   # the reference's utils package and the stub; torchvision stays loaded
            if k not in saved[4] and (k.split(".")[0] in ("utils", "matplotlib")):
                del sys.modules[k]
    assert len(models) == 1, models
    return buf.getvalue(), models[0][1], models[0][0].state_dict()


def main():
    torch.set_num_threads(1)
    out = {}
    for name, (N, Nq, D, C, seed, flags) in CASES.items():
        xtr, ytr, xte, yte = features(N, Nq, D, C, seed)
        vnames = ["v_c%d_%03d" % (int(yte[i]), i) for i in range(Nq)]
        with tempfile.TemporaryDirectory() as d:
            fd = os.path.join(d, "feature")
            os.makedirs(fd)
            for split, x, y in (("train", xtr, ytr), ("test", xte, yte)):
                torch.save(x, os.path.join(fd, "ucf101_%s_feature.pth.tar" % split))
                torch.save(y, os.path.join(fd, "ucf101_%s_label.pth.tar" % split))
            with open(os.path.join(fd, "ucf101_test_vname.pkl"), "wb") as fp:
                pickle.dump([[v] for v in vnames], fp)
            stdout, init, sd = run_reference(d, flags)
            stdout = stdout.replace(d, "<DIR>")
            with open(os.path.join(fd, "model.pth.tar-lp-ucf101-prob.json")) as fp:
                prob = json.load(fp)
        assert sorted(prob) == sorted(vnames)
        out[name + "/train_feature"], out[name + "/train_label"] = xtr.numpy(), ytr.numpy()
        out[name + "/test_feature"], out[name + "/test_label"] = xte.numpy(), yte.numpy()
        out[name + "/vname"] = np.array(vnames)
        out[name + "/flags"] = np.array(json.dumps(flags))
        out[name + "/stdout"] = np.array(stdout)
        out[name + "/prob"] = np.array([prob[v][0] for v in vnames], dtype=np.float64)
        for k, v in sd.items():
            out[name + "/state/" + k] = v.numpy()
        for k, v in init.items():
            out[name + "/init/" + k] = v.numpy()
        print(name, stdout.strip().splitlines()[-3:])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
