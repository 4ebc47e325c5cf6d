"""The reference's LMDB video datasets (dataset/lmdb_dataset.py) over `coclr_b200.lmdb_read`, without pandas.

Each class keeps the reference's name, keyword arguments, video list (`video_subset`: the rows of its pandas frame, in
order) and frame samplers with their exact random draws.  Two differences, both deliberate:
  * `root` and the database paths have no defaults: they are always passed in;
  * `__getitem__` returns the sampled frames as JPEG byte views (memoryviews into the map) in the order the reference
    hands them to its transform, with the label / source id / path as the reference returns them.  Decoding and the
    transform run on the GPU (coclr_b200.loaders).  For a 2-stream class the frames are
    rgb[:T] + flow[:T] + rgb[T:] + flow[T:].
The samplers draw from `self.rng` (np.random by default, as in the reference; a loader sets its own RandomState).
`refs(index, frame_index)` names every sampled frame as (stream, video key, frame) so that a batch can decode each
distinct frame once.
"""
import csv
import json
import os

import numpy as np

from . import lmdb_read

__all__ = [
    'UCF101LMDB_2CLIP', 'UCF101Flow_LMDB_2CLIP', 'UCF101_2STREAM_LMDB_2CLIP',
    'K400_LMDB_2CLIP', 'K400_Flow_LMDB_2CLIP', 'K400_2STREAM_LMDB_2CLIP',
    'UCF101LMDB', 'UCF101Flow_LMDB',
    'HMDB51LMDB', 'HMDB51Flow_LMDB',
]


def read_classes(root):
    """ClassInd.txt: bare names (which may hold spaces) or 'index, name' lines; the reference keeps what follows the
    last comma, stripped, when the first line has a comma."""
    with open(os.path.join(root, 'ClassInd.txt')) as f:
        classes = [line.strip() for line in f.readlines()]
    if ',' in classes[0]:
        classes = [c.split(',')[-1].strip() for c in classes]
    return classes


def read_split(path):
    """A split CSV without header: [path, frame count] per row."""
    with open(path, newline='') as f:
        return [[r[0], int(r[1])] for r in csv.reader(f) if r]


def _part(path, i):
    parts = path.split('/')
    return parts[i] if -len(parts) <= i < len(parts) else None


class _Database:
    """One opened LMDB with the reference's special keys decoded."""

    def __init__(self, path):
        self.path = path
        self.env = lmdb_read.open(path)
        self.length = self._load(b'__len__')
        self.keys = [bytes(k).decode() for k in self._load(b'__keys__')]
        self.order = [bytes(k).decode() for k in self._load(b'__order__')]
        self.video_id = dict(zip(self.order, ['%09d' % i for i in range(len(self.order))]))
        self._vlen = None

    def _load(self, key):
        v = self.env.get(key)
        if v is None:
            raise ValueError("%s: no %r key (not one of the reference's video databases)" % (self.path, key))
        return lmdb_read.unpack(v)

    @property
    def vlen(self):
        """`__vlen__` paired with `__order__` as the reference pairs them: sorted by key, then zipped with the names."""
        if self._vlen is None:
            vlen = self._load(b'__vlen__')
            ordered = [v for _, v in sorted(zip(self.keys, vlen), key=lambda x: x[0])]
            self._vlen = list(zip(self.order, ordered))
        return self._vlen

    def video(self, vname):
        """The video's frames: a list of JPEG byte views."""
        key = self.video_id[vname]
        v = self.env.get(key.encode('ascii'))
        if v is None:
            raise ValueError("%s: video %s (key %s) is missing" % (self.path, vname, key))
        return lmdb_read.unpack(v)


def _merge_vlen(rows, pairs):
    """pandas' video_info.merge(DataFrame(pairs, columns=[3, 4]), left_on=3, right_on=3).dropna(): an inner join on
    the video name in row order (each match appends the database's length), rows with a missing length dropped."""
    by_name = {}
    for name, vlen in pairs:
        by_name.setdefault(name, []).append(vlen)
    return [r + [v] for r in rows for v in by_name.get(r[3], ()) if v is not None]


def _val_subset(rows, mode):
    """mode 'val' keeps pandas' sample(frac=0.3, random_state=666) of the rows, in its order."""
    if mode != 'val':
        return rows
    pick = np.random.RandomState(666).choice(len(rows), size=round(0.3 * len(rows)), replace=False)
    return [rows[i] for i in pick]


class _LMDBVideos:
    clips = 2                   # 2: double_sampler (pre-training), 1: frame_sampler
    streams = ('rgb',)
    k400 = False

    def _setup(self, root, mode, num_frames, ds, window, return_label, return_path, return_source):
        self.root, self.mode, self.num_frames, self.ds = root, mode, num_frames, ds
        self.window = window
        self.return_label, self.return_path, self.return_source = return_label, return_path, return_source
        self.rng = np.random
        classes = read_classes(root)
        self.classes = classes
        self.num_class = len(classes)
        self.class_to_idx = {c: i for i, c in enumerate(classes)}
        self.idx_to_class = dict(enumerate(classes))

    def _ucf_rows(self, which_split):
        split_mode = 'test' if self.mode == 'val' else self.mode
        rows = read_split(os.path.join(self.root, '%s_split%02d.csv' % (split_mode, which_split)))
        rows = [[p, n, _part(p, -3), '%s/%s' % (_part(p, -3), _part(p, -2))] for p, n in rows]
        if len(set(r[2] for r in rows)) != self.num_class:
            raise ValueError("%s: the split's classes differ from ClassInd.txt" % self.root)
        return rows

    def _k400_rows(self, split_mode, full_name=False):
        rows = read_split(os.path.join(self.root, '%s_split.csv' % split_mode))
        rows = [[p, n, _part(p, -2), p if full_name else '%s/%s' % (_part(p, -2), _part(p, -1))] for p, n in rows]
        classes = set(self.classes)
        return [r for r in rows if r[2] in classes]

    def _finish(self, rows, vlen_col):
        self.vlen_col = vlen_col
        if self.k400:
            short = lambda v: v - self.num_frames * self.ds - 1 <= 0            # noqa: E731
        else:
            short = lambda v: v - self.num_frames // 2 * self.ds - 1 <= 0       # noqa: E731  max padding: half
        self.video_info = [r for r in rows if not short(r[vlen_col])]
        self.video_subset = _val_subset(self.video_info, self.mode)

    # -- samplers ----------------------------------------------------------------------------------------------------
    def frame_sampler(self, total):
        n, ds, rs = self.num_frames, self.ds, self.rng
        if self.mode == 'test' or self.window:                  # half overlap - 1
            if total - n * ds <= 0:                             # pad left, only sample once
                sequence = np.arange(n) * ds
                seq_idx = np.zeros_like(sequence)
                sequence = sequence[sequence < total]
                seq_idx[-len(sequence):] = sequence
            else:
                available = total - n * ds
                start = np.expand_dims(np.arange(0, available + 1, n * ds // 2 - 1), 1)
                seq_idx = (np.expand_dims(np.arange(n) * ds, 0) + start).flatten()
        else:                                                   # train or val
            if total - n * ds <= 0:                             # pad left
                sequence = np.arange(n) * ds + rs.choice(range(ds), 1)
                seq_idx = np.zeros_like(sequence)
                sequence = sequence[sequence < total]
                seq_idx[-len(sequence):] = sequence
            else:
                start = rs.choice(range(total - n * ds), 1)
                seq_idx = np.arange(n) * ds + start
        return seq_idx

    def double_sampler(self, total):
        return np.concatenate([self.frame_sampler(total), self.frame_sampler(total)])

    def sample(self, index):
        """The frame indices item `index` samples (the reference's draws, on self.rng)."""
        vlen = self.video_subset[index][self.vlen_col]
        return self.double_sampler(vlen) if self.clips == 2 else self.frame_sampler(vlen)

    # -- items -------------------------------------------------------------------------------------------------------
    def refs(self, index, frame_index):
        """(stream, video key, frame) of every frame in transform order: stream i of self.streams."""
        vname = self.video_subset[index][3]
        keys = [db.video_id[vname] for db in self.dbs]
        if len(keys) == 1:
            return [(0, keys[0], int(f)) for f in frame_index]
        T = self.num_frames
        fi = [int(f) for f in frame_index]
        return ([(0, keys[0], f) for f in fi[:T]] + [(1, keys[1], f) for f in fi[:T]] +
                [(0, keys[0], f) for f in fi[T:]] + [(1, keys[1], f) for f in fi[T:]])

    def label(self, index):
        return self.class_to_idx[self.video_subset[index][2]]

    def source_id(self, index):
        vname = self.video_subset[index][3]
        return self.video_source[vname if self.k400 else vname.split('/')[-1][:-4]]

    def frames(self, index, frame_index):
        """JPEG byte views of the sampled frames in transform order."""
        vname = self.video_subset[index][3]
        videos = [db.video(vname) for db in self.dbs]
        out = []
        for s, _, f in self.refs(index, frame_index):
            if not 0 <= f < len(videos[s]):
                raise ValueError("%s: video %s has %d frames, frame %d was sampled" % (
                    self.dbs[s].path, vname, len(videos[s]), f))
            out.append(videos[s][f])
        return out

    def __getitem__(self, index):
        frames = self.frames(index, self.sample(index))
        return self._returns(index, frames)

    def _returns(self, index, frames):
        if not self.return_label:
            return frames
        vid, vpath = self.label(index), self.video_subset[index][0]
        if self.return_source:
            return frames, self.source_id(index), vid
        if self.return_path:
            return frames, (vid, vpath)
        return frames, vid

    def __len__(self):
        return len(self.video_subset)

    def encode_action(self, action_name):
        return self.class_to_idx[action_name]

    def decode_action(self, action_code):
        return self.idx_to_class[action_code]


class UCF101LMDB_2CLIP(_LMDBVideos):
    def __init__(self, root, db_path, mode='val', num_frames=32, ds=1, which_split=1, window=False,
                 return_path=False, return_label=False, return_source=False):
        self._setup(root, mode, num_frames, ds, window, return_label, return_path, return_source)
        self.which_split, self.db_path = which_split, db_path
        self.dbs = [_Database(db_path)]
        rows = self._ucf_rows(which_split)
        if return_source:
            self.video_source = _read_json(os.path.join(root, 'video_source.json'))
        self._finish(rows, 1)


class UCF101LMDB(UCF101LMDB_2CLIP):
    clips = 1


class HMDB51LMDB(UCF101LMDB):
    pass


class UCF101Flow_LMDB_2CLIP(_LMDBVideos):
    def __init__(self, root, db_path, mode='val', num_frames=32, ds=1, which_split=1,
                 return_label=False, return_path=False, return_source=False):
        self._setup(root, mode, num_frames, ds, False, return_label, return_path, return_source)
        self.which_split, self.db_path = which_split, db_path
        self.dbs = [_Database(db_path)]
        rows = self._ucf_rows(which_split)
        if return_source:
            self.video_source = _read_json(os.path.join(root, 'video_source.json'))
        self._finish(_merge_vlen(rows, self.dbs[0].vlen), 4)   # flow may have another frame count than rgb


class UCF101Flow_LMDB(UCF101Flow_LMDB_2CLIP):
    clips = 1


class HMDB51Flow_LMDB(UCF101Flow_LMDB):
    pass


def _two_stream_vlen(rgb, flow):
    names = set(rgb.order)
    return [(n, v) for n, v in flow.vlen if n in names]


class UCF101_2STREAM_LMDB_2CLIP(_LMDBVideos):
    streams = ('rgb', 'flow')

    def __init__(self, root, db_path_flow, db_path_rgb, mode='val', num_frames=32, ds=1, which_split=1,
                 return_label=False, return_path=False, return_source=False):
        self._setup(root, mode, num_frames, ds, False, return_label, return_path, return_source)
        self.which_split, self.db_path_flow, self.db_path_rgb = which_split, db_path_flow, db_path_rgb
        rgb, flow = _Database(db_path_rgb), _Database(db_path_flow)
        self.dbs = [rgb, flow]
        rows = self._ucf_rows(which_split)
        self.video_source = _read_json(os.path.join(root, 'video_source.json'))
        rows = [r[:4] + [min(r[1], r[4])] for r in _merge_vlen(rows, _two_stream_vlen(rgb, flow))]
        self._finish(rows, 4)

    def _returns(self, index, frames):
        if self.return_source:
            if self.return_label:
                return frames, self.source_id(index), self.label(index)
            return frames, self.source_id(index)
        return frames


class _Kinetics(_LMDBVideos):
    k400 = True

    def _returns(self, index, frames):
        if not self.return_label:
            return frames
        if self.return_path:
            return frames, (self.label(index), self.video_subset[index][0])
        return frames, self.label(index)


class KineticsLMDB_2CLIP(_Kinetics):
    def __init__(self, root, db_path, filename, mode='val', num_frames=32, ds=1, window=False,
                 return_label=False, return_path=False, is_flow=False):
        self._setup(root, mode, num_frames, ds, window, return_label, return_path, False)
        split_mode = 'val' if mode == 'test' else mode
        self.db_path = os.path.join(db_path, '%s_%s.lmdb' % (filename, split_mode))
        self.is_flow = is_flow
        self.dbs = [_Database(self.db_path)]
        rows = self._k400_rows(split_mode)
        self.video_source = _read_json(os.path.join(root, 'video_source.json'))
        if is_flow:
            rows = _merge_vlen(rows, self.dbs[0].vlen)
        self._finish(rows, 4 if is_flow else 1)


class K400_LMDB_2CLIP(KineticsLMDB_2CLIP):
    def __init__(self, root, db_path, filename='k400_frame', **kwargs):
        super().__init__(root=root, db_path=db_path, filename=filename, is_flow=False, **kwargs)


class K400_Flow_LMDB_2CLIP(KineticsLMDB_2CLIP):
    def __init__(self, root, db_path, filename='k400_tvl1_frame', **kwargs):
        super().__init__(root=root, db_path=db_path, filename=filename, is_flow=True, **kwargs)


class Kinetics_2STREAM_LMDB_2CLIP(_Kinetics):
    streams = ('rgb', 'flow')

    def __init__(self, root, db_path_flow, db_path_rgb, filename_flow, filename_rgb, mode='val', num_frames=32, ds=1,
                 return_label=False, return_path=False, return_source=False):
        self._setup(root, mode, num_frames, ds, False, return_label, return_path, return_source)
        split_mode = 'val' if mode == 'test' else mode
        self.db_path_flow = os.path.join(db_path_flow, '%s_%s.lmdb' % (filename_flow, split_mode))
        self.db_path_rgb = os.path.join(db_path_rgb, '%s_%s.lmdb' % (filename_rgb, split_mode))
        rgb, flow = _Database(self.db_path_rgb), _Database(self.db_path_flow)
        self.dbs = [rgb, flow]
        rows = self._k400_rows(split_mode, full_name=True)
        self.video_source = _read_json(os.path.join(root, 'video_source.json'))
        if rows and len(rows[0][3].split('/')) != 2:             # long path to short path
            for r in rows:
                r[3] = '/'.join(r[3].split('/')[-2:])
        rows = [r[:4] + [min(r[1], r[4])] for r in _merge_vlen(rows, _two_stream_vlen(rgb, flow))]
        self._finish(rows, 4)

    _returns = UCF101_2STREAM_LMDB_2CLIP._returns


class K400_2STREAM_LMDB_2CLIP(Kinetics_2STREAM_LMDB_2CLIP):
    def __init__(self, root, db_path_flow, db_path_rgb, filename_flow='k400_tvl1_frame', filename_rgb='k400_frame',
                 **kwargs):
        super().__init__(root=root, db_path_flow=db_path_flow, db_path_rgb=db_path_rgb,
                         filename_flow=filename_flow, filename_rgb=filename_rgb, **kwargs)


def _read_json(path):
    with open(path) as f:
        return json.load(f)
