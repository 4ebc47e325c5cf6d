"""Writes tests/golden/two_stream.npz by running the UNMODIFIED reference eval/merge_2stream_prob.py ($COCLR_REFERENCE)
on the CPU: its merge_prob (--mode c) over seeded probability JSON files and its merge_sim (--mode s) over seeded
feature directories.

The script is imported as it is, with three shims, each plumbing: a stub `matplotlib` (imported, not used), `np.int =
int` (removed in NumPy 1.24), and the module's `__file__` pointed into a temporary tree so that get_action_idx reads
this file's class list from process_data/data/<dataset>_beegfs/ClassInd.txt.  Its sys.exit() is caught.  Two functions
are wrapped to record what passes through them, unchanged: get_action_idx's class list and preprocess's inputs (the
four aligned feature sets, from which the reference's alignment order is recovered row by row).

Mode c cases: UCF101-style vnames (.../frame/<Action>/v_<Action>_gXX_cYY/) with a 'N,Action' class list, HMDB51-style
ones with a plain list, and k400-style ones (.../<action>/<id>, action at [-2], names with spaces); both JSON value
formats ({'mean_prob': [[...]]} and plain lists, nested or flat); rows where p1, p2 or the fused mean tie between
classes.  Mode s cases: stream 1 or stream 2 has more train videos (either isin branch), both branches run, or neither;
D1 != D2 (some not multiples of 4) and Nk not a multiple of 4.  For each retrieval case the seed is the first whose
smallest float64 similarity gap at every k boundary (k-th vs (k+1)-th most similar item of any query) is above 1e-4,
far above fp32 error, so the top-k sets are the same in any faithful fp32 evaluation; the gaps are stored.

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_two_stream.py
"""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402

OUT = os.path.join(HERE, "two_stream.npz")
KS = (1, 5, 10, 20, 50)
GAP_MIN = 1e-4

# mode c: name -> (dataset, class-list style, n videos, classes, value formats of stream 1 / 2, seed)
PROB_CASES = {
    "ucf": ("ucf101", "comma", 64, 12, ("dict", "nested"), 3),
    "hmdb": ("hmdb51", "plain", 45, 9, ("nested", "dict"), 4),
    "k400": ("k400", "plain", 50, 10, ("flat", "dict"), 5),
}
# mode s: name -> (n train 1, n train 2, n test 1, n test 2, names only stream 1 / 2 has, D1, D2, classes)
SIM_CASES = {
    "filter1": (70, 63, 37, 33, 0, 40, 24, 7),      # stream 1 longer: stream 1 is filtered
    "filter2": (66, 75, 30, 34, 0, 30, 18, 6),      # stream 2 longer: stream 2 is filtered
    "both": (66, 70, 31, 33, 4, 64, 36, 8),         # stream 2 filtered, then still shorter: stream 1 filtered too
    "equal": (61, 61, 29, 29, 0, 36, 36, 5),
}


def load_reference(tmp):
    spec = importlib.util.spec_from_file_location("merge_2stream_prob_ref", os.path.join(REF, "eval",
                                                                                         "merge_2stream_prob.py"))
    mod = importlib.util.module_from_spec(spec)
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot.switch_backend = lambda *a, **k: None
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    np.int = int
    sys.path.insert(0, REF)
    spec.loader.exec_module(mod)
    os.makedirs(os.path.join(tmp, "a", "b"))
    mod.__file__ = os.path.join(tmp, "a", "b", "merge_2stream_prob.py")   # ../../process_data/data -> tmp
    return mod


def run(fn, args):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        try:
            fn(args)
        except SystemExit:
            pass
    return buf.getvalue()


# ---------------------------------------------------------------------------------------------------------------------
# mode c
# ---------------------------------------------------------------------------------------------------------------------
def class_names(dataset, C, rng):
    if dataset == "k400":
        base = ["abseiling", "air drumming", "baking cookies", "cartwheeling", "dancing ballet", "eating chips",
                "folding napkins", "golf putting", "hula hooping", "juggling balls", "kicking soccer ball"]
    else:
        base = ["ApplyEyeMakeup", "Archery", "BabyCrawling", "Basketball", "CliffDiving", "Drumming", "Fencing",
                "HammerThrow", "Hammering", "JumpRope", "Kayaking", "PlayingCello", "Rowing"]
    names = list(base[:C])
    rng.shuffle(names)               # class order is the list's, not alphabetical
    return names


def vname_of(dataset, action, i):
    if dataset == "k400":
        return "/data/k400/val_256/%s/yt%06d_%06d_%06d" % (action, 1000 + 7 * i, 10 * i, 10 * i + 10)
    if dataset == "hmdb51":
        return "/data/hmdb51/frame/%s/%s_vid%03d_f_cm_np1_fr_med_%d/" % (action, action.lower(), i, i % 3)
    return "/data/ucf101/frame/%s/v_%s_g%02d_c%02d/" % (action, action, 8 + i % 17, 1 + i % 5)


def prob_case(dataset, style, N, C, formats, seed):
    rng = np.random.default_rng(seed)
    names = class_names(dataset, C, rng)
    labels = rng.integers(0, C, N)
    vnames = [vname_of(dataset, names[c], i) for i, c in enumerate(labels)]

    def softmax(z):
        e = np.exp(z - z.max(1, keepdims=True))
        return e / e.sum(1, keepdims=True)

    onehot = np.eye(C)[labels]
    p1 = softmax(rng.normal(size=(N, C)) * 1.5 + 1.2 * onehot)
    p2 = softmax(rng.normal(size=(N, C)) * 1.5 + 1.2 * onehot)
    for r in range(0, N, 5):          # ties: the target and another class share the top value, either side of it
        t, o = int(labels[r]), int(rng.integers(0, C))
        if o == t:
            o = (t + 1) % C
        kind = (r // 5) % 3
        if kind == 0:                 # p1 ties
            p1[r, t] = p1[r, o] = p1[r].max() + 0.25
        elif kind == 1:               # p2 ties
            p2[r, t] = p2[r, o] = p2[r].max() + 0.25
        else:                         # only the fused mean ties: (a + b) / 2 at t and at o
            p1[r, t], p1[r, o] = 0.875, 0.625
            p2[r, t], p2[r, o] = 0.625, 0.875
    lines = ["%d,%s" % (i + 1, n) for i, n in enumerate(names)] if style == "comma" else list(names)
    class_text = "\n".join(lines) + "\n"

    def dump(p, fmt):
        if fmt == "dict":
            return json.dumps({v: {"mean_prob": [row.tolist()]} for v, row in zip(vnames, p)})
        if fmt == "nested":
            return json.dumps({v: [row.tolist()] for v, row in zip(vnames, p)})
        return json.dumps({v: row.tolist() for v, row in zip(vnames, p)})

    order = rng.permutation(N)        # stream 2's file lists the videos in another order
    j1 = dump(p1, formats[0])
    d2 = json.loads(dump(p2, formats[1]))
    j2 = json.dumps({vnames[i]: d2[vnames[i]] for i in order})
    return dict(class_text=class_text, json1=j1, json2=j2, p1=p1, p2=p2, labels=labels, vnames=vnames)


def make_prob(mod, tmp, name, spec):
    dataset, style, N, C, formats, seed = spec
    c = prob_case(dataset, style, N, C, formats, seed)
    d = os.path.join(tmp, "process_data", "data", "%s_beegfs" % dataset)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "ClassInd.txt"), "w") as f:
        f.write(c["class_text"])
    for i in (1, 2):
        with open(os.path.join(tmp, "%s_%d.json" % (name, i)), "w") as f:
            f.write(c["json%d" % i])
    seen = []
    orig = mod.get_action_idx
    mod.get_action_idx = lambda ds: seen.append(orig(ds)) or seen[-1]
    try:
        out = run(mod.merge_prob, argparse.Namespace(prob1=os.path.join(tmp, "%s_1.json" % name),
                                                      prob2=os.path.join(tmp, "%s_2.json" % name),
                                                      dataset=dataset, mode="c"))
    finally:
        mod.get_action_idx = orig
    return {"dataset": np.array(dataset), "class_text": np.array(c["class_text"]), "json1": np.array(c["json1"]),
            "json2": np.array(c["json2"]), "p1": c["p1"], "p2": c["p2"], "label": c["labels"],
            "vname": np.array(c["vnames"]), "action_list": np.array(seen[0]), "stdout": np.array(out)}


# ---------------------------------------------------------------------------------------------------------------------
# mode s
# ---------------------------------------------------------------------------------------------------------------------
def sim_case(spec, seed):
    n1tr, n2tr, n1te, n2te, extra, D1, D2, ncls = spec
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)

    def names(split, n_common, n1_only):
        common = ["/data/ucf101/frame/A%d/v_%s_g%02d_c%02d/" % (i % ncls, split, i, i % 7) for i in range(n_common)]
        only = ["/data/ucf101/frame/A%d/v_%s_only_%02d/" % (i % ncls, split, i) for i in range(n1_only)]
        return common, only

    sets = {}
    for split, n1, n2 in (("train", n1tr, n2tr), ("test", n1te, n2te)):
        common, only1 = names(split, min(n1, n2) - extra, extra)
        v1 = common + only1 + (["/data/ucf101/frame/A0/v_%s_s1_%02d/" % (split, i) for i in range(n1 - len(common)
                                                                                                   - extra)])
        v2 = common + (["/data/ucf101/frame/A0/v_%s_s2_%02d/" % (split, i) for i in range(n2 - len(common))])
        sets[split] = [list(rng.permutation(v1)), list(rng.permutation(v2))]
    centers1, centers2 = torch.randn(ncls, D1, generator=g), torch.randn(ncls, D2, generator=g)
    out = {}
    for split in ("train", "test"):
        for s, (centers, D) in enumerate(((centers1, D1), (centers2, D2))):
            vn = sets[split][s]
            lab = torch.tensor([int(v.split("/")[-3][1:]) for v in vn])
            feat = (centers[lab] + 2.5 * torch.randn(len(vn), D, generator=g) + 0.4).float()
            out[split, s] = (vn, feat, lab)
    return out


def boundary_gaps(sim):
    s = np.sort(sim, axis=1)[:, ::-1]
    return np.array([float((s[:, k - 1] - s[:, k]).min()) if k < s.shape[1] else np.inf for k in KS])


def make_sim(mod, tmp, name, spec):
    for seed in range(100 * (list(SIM_CASES).index(name) + 1), 100 * (list(SIM_CASES).index(name) + 2)):
        data = sim_case(spec, seed)
        d1, d2 = os.path.join(tmp, name, "s%d_1" % seed), os.path.join(tmp, name, "s%d_2" % seed)
        for s, d, prefix in ((0, d1, "ucf101"), (1, d2, "ucf101-f")):
            os.makedirs(d)
            for split in ("train", "test"):
                vn, feat, lab = data[split, s]
                torch.save(feat, os.path.join(d, "%s_%s_feature.pth.tar" % (prefix, split)))
                torch.save(lab, os.path.join(d, "%s_%s_label.pth.tar" % (prefix, split)))
                with open(os.path.join(d, "%s_%s_vname.pkl" % (prefix, split)), "wb") as fp:
                    pickle.dump([[v] for v in vn], fp)
        seen = []
        orig = mod.preprocess
        mod.preprocess = lambda t: seen.append(t.clone()) or orig(t)
        try:
            out = run(mod.merge_sim, argparse.Namespace(prob1=d1, prob2=d2, dataset="ucf101", mode="s"))
        finally:
            mod.preprocess = orig
        tr1, tr2, te1, te2 = seen      # the reference's call order
        order = {}
        for key, aligned, (split, s) in (("train1", tr1, ("train", 0)), ("train2", tr2, ("train", 1)),
                                         ("test1", te1, ("test", 0)), ("test2", te2, ("test", 1))):
            rows = {r.numpy().tobytes(): i for i, r in enumerate(data[split, s][1])}
            order[key] = np.array([rows[r.numpy().tobytes()] for r in aligned], dtype=np.int64)
        q1, k1 = (F.normalize(x.double() - x.double().mean(0), dim=1) for x in (te1, tr1))
        q2, k2 = (F.normalize(x.double() - x.double().mean(0), dim=1) for x in (te2, tr2))
        gaps = boundary_gaps((q1 @ k1.t() + q2 @ k2.t()).numpy())
        if gaps.min() > GAP_MIN:
            break
    else:
        raise RuntimeError("no seed with k-boundary gaps above %g for %s" % (GAP_MIN, name))
    res = {"seed": np.array(seed), "stdout": np.array(out), "gaps": gaps}
    for split in ("train", "test"):
        for s in (0, 1):
            vn, feat, lab = data[split, s]
            res["%s%d/vname" % (split, s + 1)] = np.array(vn)
            res["%s%d/feature" % (split, s + 1)] = feat.numpy()
            res["%s%d/label" % (split, s + 1)] = lab.numpy()
    for k, v in order.items():
        res["order_" + k] = v
    return res


def main():
    torch.set_num_threads(1)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        mod = load_reference(tmp)
        for name, spec in PROB_CASES.items():
            for k, v in make_prob(mod, tmp, name, spec).items():
                out["prob/%s/%s" % (name, k)] = v
            print(name, out["prob/%s/stdout" % name].item().strip().splitlines())
        for name, spec in SIM_CASES.items():
            r = make_sim(mod, tmp, name, spec)
            for k, v in r.items():
                out["sim/%s/%s" % (name, k)] = v
            print(name, "seed", int(r["seed"]), "gaps", r["gaps"], r["stdout"].item().strip().splitlines())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
