"""Writes tests/golden/reference_cli.npz from the UNMODIFIED reference ($COCLR_REFERENCE): the options of its
main_nce.py / main_coclr.py, and its multi_nce_loss (main_coclr.py:343-346) and UberNCE loss lines (main_nce.py:321-322)
on three seeded inputs, executed from its source text."""
import ast
import json
import os
import re
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402

OUT = os.path.join(HERE, "reference_cli.npz")


def ref_flags(path):
    out = {}
    for m in re.finditer(r"add_argument\(([^)]*)\)", open(path).read()):
        names = re.findall(r"'(-{1,2}[\w-]+)'", m.group(1))
        takes_value = "store_true" not in m.group(1)
        nargs2 = "nargs=2" in m.group(1)
        for n in names:
            out[n] = [takes_value, nargs2]
    return out


def loss_inputs():
    """The seeded (logits, mask) pairs tests/test_host_cpu.py feeds both implementations."""
    g = torch.Generator().manual_seed(9)
    pairs = []
    for _ in range(3):
        logits = torch.randn(6, 1 + 40, generator=g) * 4
        mask = torch.rand(6, 41, generator=g) < 0.15
        mask[:, 0] = True
        pairs.append((logits, mask))
    return pairs


def main():
    flags = {"main_nce": ref_flags(os.path.join(REF, "main_nce.py")),
             "main_coclr": ref_flags(os.path.join(REF, "main_coclr.py"))}
    src = open(os.path.join(REF, "main_coclr.py")).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "multi_nce_loss"][0]
    ns = {"torch": torch, "F": F}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "ref_multi_nce_loss", "exec"), ns)
    lines = open(os.path.join(REF, "main_nce.py")).read().splitlines()
    uber = [ln.strip() for ln in lines if ln.strip().startswith("loss = - (F.log_softmax(output, dim=1) * target)")]
    assert len(uber) == 1
    out = {"flags_json": np.array(json.dumps(flags, sort_keys=True))}
    # --pretrain A B: the merge of the two checkpoints and the renames of B's query encoder (main_coclr.py:250-302)
    out["two_checkpoint_merge"] = np.array(["state_dict = {**first_dict, **second_dict}" in src,
                                            "k = k.replace('encoder_q.', 'encoder_k.')" in src,
                                            "k.replace('encoder_q.', 'sampler.')" in src])
    for i, (logits, mask) in enumerate(loss_inputs()):
        out["multi_nce_loss/%d" % i] = ns["multi_nce_loss"](logits, mask).detach().numpy()
        env = {"F": F, "output": logits, "target": mask}
        exec(uber[0], env)
        out["ubernce_loss/%d" % i] = env["loss"].mean().detach().numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
