"""Writes tests/golden/datasets.npz by running the UNMODIFIED reference dataset/lmdb_dataset.py ($COCLR_REFERENCE)
on the seeded fixture of tests/tools/dataset_fixture.py, with a dict-backed stand-in for the `lmdb` package and
`msgpack.loads` given msgpack 0.6.2's semantics (raw=True: str-family values come back as bytes).

  pool_data, pool_off   the fixture's JPEG pool (every frame of every database is one of these)
  subsets               JSON: {"<class> <mode> ds<ds>": video_subset rows (the pandas frame's rows, in order)}
  samples               JSON: {"<class> <mode> ds<ds>": [frame indices of __getitem__(i) for every i]}, after
                        np.random.seed(SAMPLE_SEED)
  out_<case>, idx_<case>   the reference's transformed batch (DataLoader, num_workers=0, over the items idx_<case>,
                        seeded with torch.manual_seed / np.random.seed / random.seed(TRANSFORM_SEED) after the
                        iterator is made):  nce (UCF101LMDB_2CLIP, main_nce's get_transform), coclr
                        (UCF101_2STREAM_LMDB_2CLIP, main_coclr's), clf (UCF101LMDB, main_classifier's 'train' recipe,
                        before the batch flip), and the test views test50 (centre) and test21 (five-crop corner 2,
                        flipped): UCF101LMDB mode 'test' through test_10crop's transform, one video per batch, stored
                        as uint8 (the float output * 255, exact) [3, sum of len_<case>, D, D]

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_datasets.py
"""
import functools
import importlib.util
import json
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
from make_golden import REF  # noqa: E402
import dataset_fixture as F  # noqa: E402

OUT = os.path.join(HERE, "datasets.npz")
NF = 4                      # num_frames of every case
SAMPLE_SEED, TRANSFORM_SEED = 123, 7
IMG = 16                    # img_dim of the pre-training cases (the classifier recipe's is make_golden_clf_augment.D)

UCF_CLASSES = ["UCF101LMDB_2CLIP", "UCF101LMDB", "HMDB51LMDB", "UCF101Flow_LMDB_2CLIP", "UCF101Flow_LMDB",
               "HMDB51Flow_LMDB", "UCF101_2STREAM_LMDB_2CLIP"]
K400_CLASSES = ["K400_LMDB_2CLIP", "K400_Flow_LMDB_2CLIP", "K400_2STREAM_LMDB_2CLIP"]


def class_kwargs(name, data, split, mode, ds):
    """The keyword arguments both sides take for `name` on the fixture at data / split."""
    kw = dict(mode=mode, num_frames=NF, ds=ds)
    if name.startswith("HMDB"):
        kw["root"] = os.path.join(split, "hmdb51")
    elif name.startswith("UCF"):
        kw["root"] = os.path.join(split, "ucf101")
    else:
        kw["root"] = os.path.join(split, "k400")
    if name in ("UCF101LMDB_2CLIP", "UCF101LMDB"):
        kw["db_path"] = os.path.join(data, F.RGB)
    elif name in ("UCF101Flow_LMDB_2CLIP", "UCF101Flow_LMDB"):
        kw["db_path"] = os.path.join(data, F.FLOW)
    elif name == "HMDB51LMDB":
        kw["db_path"] = os.path.join(data, F.HRGB)
    elif name == "HMDB51Flow_LMDB":
        kw["db_path"] = os.path.join(data, F.HFLOW)
    elif name == "UCF101_2STREAM_LMDB_2CLIP":
        kw["db_path_rgb"], kw["db_path_flow"] = os.path.join(data, F.RGB), os.path.join(data, F.FLOW)
    elif name == "K400_LMDB_2CLIP":
        kw["db_path"] = os.path.join(data, os.path.dirname(F.KRGB))
    elif name == "K400_Flow_LMDB_2CLIP":
        kw["db_path"] = os.path.join(data, os.path.dirname(F.KFLOW))
    else:
        kw["db_path_rgb"] = os.path.join(data, os.path.dirname(F.KRGB))
        kw["db_path_flow"] = os.path.join(data, os.path.dirname(F.KFLOW))
    if "2STREAM" in name:
        kw["return_source"] = True
        kw["return_label"] = True
    return kw


def cases():
    """(class, mode, ds, window) of every recorded subset / sampler case."""
    out = []
    for name in UCF_CLASSES + K400_CLASSES:
        for mode in ("train", "val", "test"):
            if name == "K400_LMDB_2CLIP" and mode != "train":
                continue                             # its val database lacks a video of the CSV
            for ds in (1, 2):
                out.append((name, mode, ds, False))
    return out + [("UCF101LMDB_2CLIP", "train", 1, True), ("UCF101LMDB", "val", 2, True)]


# (case, (aug_idx, flip_idx), test-split items): the centre view, and a flipped five-crop corner
TEST_VIEWS = [("test50", (5, 0), [5, 0, 1, 2]), ("test21", (2, 1), [1, 5, 3])]


def case_key(name, mode, ds, window):
    return "%s %s ds%d%s" % (name, mode, ds, " window" if window else "")


def rows_json(rows):
    return [[v.item() if hasattr(v, "item") else v for v in r] for r in rows]


class _Flat(np.ndarray):
    def flatten(self, order="C"):
        # the reference's test sampler calls flatten(0); numpy < 1.x read a falsy non-string order as 'C', today's
        # numpy raises
        return np.ndarray.flatten(self, "C" if order == 0 else order)


class OldNumpy:
    """numpy for the reference module, with expand_dims results that accept flatten(0)."""

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def expand_dims(a, axis):
        return np.expand_dims(a, axis).view(_Flat)


def fake_lmdb(dbs):
    """lmdb.open(path, ...) over {path: {key: value}}."""
    class Txn:
        def __init__(self, d):
            self.d = d

        def get(self, k):
            return self.d.get(k)

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    class Env:
        def __init__(self, d):
            self.d = d

        def begin(self, write=False):
            return Txn(self.d)

    mod = types.ModuleType("lmdb")
    mod.open = lambda path, **kw: Env(dbs[os.path.normpath(path)])
    return mod


def main():
    import msgpack
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import lmdb_writer as W
    jpegs = F.pool()
    sp = F.spec()
    tmp = tempfile.mkdtemp()
    data, split = os.path.join(tmp, "data"), os.path.join(tmp, "split")
    for rel, text in sp["files"].items():
        p = os.path.join(split, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(text)
    dbs = {}
    for rel, db in sp["dbs"].items():                # the values msgpack 0.6.2's dumps wrote: byte strings as str
        vid = {n: "%09d" % i for i, n in enumerate(db["order"])}
        names = sorted(db["videos"])
        d = {vid[n].encode(): W.pack([jpegs[i] for i in db["videos"][n]], False) for n in names}
        d[b"__keys__"] = W.pack([vid[n].encode() for n in names], False)
        d[b"__len__"] = W.pack(len(names), False)
        d[b"__order__"] = W.pack([n.encode() for n in db["order"]], False)
        d[b"__vlen__"] = W.pack([len(db["videos"][n]) for n in names], False)
        dbs[os.path.normpath(os.path.join(data, rel))] = d
    sys.modules["lmdb"] = fake_lmdb(dbs)
    msgpack.loads = functools.partial(msgpack.unpackb, raw=True)
    spec = importlib.util.spec_from_file_location("reference_lmdb_dataset", os.path.join(REF, "dataset",
                                                                                          "lmdb_dataset.py"))
    L = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(L)
    L.np = OldNumpy()

    def make(name, mode, ds, **extra):
        kw = class_kwargs(name, data, split, mode, ds)
        kw.update(extra)
        if name.startswith("K400") and not name.startswith("K400_2"):
            kw.pop("return_source", None)
        return getattr(L, name)(transform=lambda seq: [torch.zeros(1)] * len(seq), **kw)

    subsets, samples = {}, {}
    for name, mode, ds, window in cases():
        key = case_key(name, mode, ds, window)
        d = make(name, mode, ds, **({"window": True} if window else {}))
        subsets[key] = rows_json(d.video_subset.itertuples(index=False))
        calls = []
        orig = d.frame_sampler
        d.frame_sampler = lambda total, orig=orig: calls.append(orig(total)) or calls[-1]   # double_sampler calls it
        np.random.seed(SAMPLE_SEED)
        per = []
        for i in range(len(d)):
            del calls[:]
            d[i]
            per.append(np.concatenate(calls).tolist())
        samples[key] = per

    # transformed batches
    from make_golden_augment import get_transform, load_reference_augmentation
    import make_golden_clf_augment as CA
    A = load_reference_augmentation()
    res = {}
    tf_nce = get_transform(A, NF, IMG)
    tf_coclr = get_transform(A, 2 * NF, IMG)
    Acl = CA.load("utils/augmentation.py", "reference_augmentation")
    Tt = CA.load("utils/transforms.py", "reference_transforms")
    for case, name, tf, idx in (("nce", "UCF101LMDB_2CLIP", tf_nce, [3, 0, 5]),
                                ("coclr", "UCF101_2STREAM_LMDB_2CLIP", tf_coclr, [2, 4, 0]),
                                ("clf", "UCF101LMDB", CA.recipe(Acl, Tt, "train"), [1, 4, 2])):
        kw = class_kwargs(name, data, split, "train", 1)
        if name != "UCF101_2STREAM_LMDB_2CLIP":
            kw["return_label"] = True
        d = getattr(L, name)(transform=tf, **kw)
        loader = torch.utils.data.DataLoader(d, batch_size=len(idx), sampler=idx, num_workers=0)
        it = iter(loader)
        torch.manual_seed(TRANSFORM_SEED)
        np.random.seed(TRANSFORM_SEED)
        random.seed(TRANSFORM_SEED)
        b = next(it)
        if case == "coclr":
            (s1, s2), target, _ = b
            out = torch.stack([s1, s2])
        else:
            out, target = b
        res["out_" + case] = out.numpy().astype(np.float32)
        res["idx_" + case] = np.array(idx, np.int64)
        res["target_" + case] = np.asarray(target, np.int64)
    from make_golden_augment import as_u8
    for case, view, idx in TEST_VIEWS:                # test_10crop's views, one video per DataLoader batch
        kw = class_kwargs("UCF101LMDB", data, split, "test", 1)
        d = L.UCF101LMDB(transform=CA.recipe(Acl, Tt, "test", view), return_label=True, **kw)
        loader = torch.utils.data.DataLoader(d, batch_size=1, sampler=idx, num_workers=0)
        it = iter(loader)
        torch.manual_seed(TRANSFORM_SEED)
        np.random.seed(TRANSFORM_SEED)
        random.seed(TRANSFORM_SEED)
        outs, lens, targets = [], [], []
        for seq, target in it:
            outs.append(as_u8(seq[0]))                 # [3, windows * NF, D, D]
            lens.append(seq.shape[2])
            targets.append(int(target))
        res["out_" + case] = np.concatenate(outs, 1)
        res["len_" + case] = np.array(lens, np.int64)
        res["idx_" + case] = np.array(idx, np.int64)
        res["target_" + case] = np.array(targets, np.int64)
    pd, po = F.pool_to_arrays(jpegs)
    np.savez_compressed(OUT, pool_data=pd, pool_off=po, subsets=np.array(json.dumps(subsets)),
                        samples=np.array(json.dumps(samples)), **res)
    print("wrote", OUT, {k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    main()
