# -*-coding:utf-8 -*-
"""On-disk batch format + input pipeline (SURVEY §8(f) rank 1): the TFRecord-free replacement of the reference's
`dump_tfrecord` (data/base_preprocess.py:229-253) and `NerDataset.build_input_fn` (dataset.py:39-55).

A `.nerrec` file is a column store of ONE split of one dataset, already padded to `max_seq_len` exactly as the
reference's tf.train.Example records are (same feature names, data/base_preprocess.py:36-71):

    bytes 0..7    magic  b'NERREC01'
    bytes 8..15   little-endian u64: length H of the JSON header
    bytes 16..    JSON header {n, max_seq_len, columns: [{name, kind, dtype, shape, offset, nbytes}, ...]}
    then          the column blobs, each 64-byte aligned, offsets relative to the start of the file

  kind 'array'   : a C-contiguous [n, ...] array of `dtype` (ids are stored in the narrowest integer type that holds
                   them and widened to int32 on read — the cast dataset.py:23-27 applies to the int64 TFRecord fields)
  kind 'strings' : [n, max_seq_len] UTF-8 strings ('tokens' / 'labels', which stay on the host).  A row is stored up to
                   its last non-'[PAD]' entry (format_sequence pads with that literal, data/base_preprocess.py:164-177):
                   `name` = u32 row pointers [n+1] into `name.len` (u8 byte length of every stored entry) and
                   `name.bytes` (the entries back to back)

A batch is a row slice of every column: the file is memory-mapped, so a batch costs one copy into (pinned) host
memory and no parsing — the per-example protobuf decode of the reference's input_fn does not exist here.
"""
import json
import os
import pickle
from collections import OrderedDict

import numpy as np
import torch

MAGIC = b'NERREC01'
_ALIGN = 64
# features that travel to the device (dataset.py:21-37) and the dtype build_graph receives them in
DEVICE_INT = ('token_ids', 'mask', 'segment_ids', 'label_ids', 'seq_len', 'softword_ids', 'bichar_ids', 'softlexicon_ids',
              'task_ids', 'lattice_ids', 'lattice_lens', 'label_mask', 'word_start')
DEVICE_FLOAT = ('softlexicon_weights', 'ex_softword_ids')
STRING_COLS = ('tokens', 'labels')
PAD_STRING = '[PAD]'


def _narrow(a):
    a = np.asarray(a)
    if a.dtype.kind in 'iu':
        lo, hi = (int(a.min()), int(a.max())) if a.size else (0, 0)
        for dt in (np.uint8, np.int16, np.int32):
            if np.iinfo(dt).min <= lo and hi <= np.iinfo(dt).max:
                return np.ascontiguousarray(a.astype(dt))
        raise ValueError('integer feature does not fit int32')
    return np.ascontiguousarray(a.astype(np.float32))


def write_records(path, features, max_seq_len):
    """features: list of per-sentence feature dicts (BasicProc.build_feature output) -> one .nerrec file."""
    n = len(features)
    cols, blobs = [], []

    def add(name, kind, arr):
        cols.append({'name': name, 'kind': kind, 'dtype': arr.dtype.str, 'shape': list(arr.shape)})
        blobs.append(arr)

    keys = [k for k in features[0] if k not in ('label_len',)] if n else []
    for k in keys:
        if k in STRING_COLS:
            rowptr, lens, chunks = np.zeros(n + 1, np.uint32), [], []
            for i, f in enumerate(features):
                row = list(f[k])
                assert len(row) == max_seq_len, k
                while row and row[-1] == PAD_STRING:
                    row.pop()
                enc = [x.encode('utf-8') for x in row]
                lens.extend(len(b) for b in enc)
                chunks.append(b''.join(enc))
                rowptr[i + 1] = rowptr[i] + len(enc)
            assert max(lens, default=0) < 256
            add(k, 'strings', rowptr)
            add(k + '.len', 'bytes', np.asarray(lens, np.uint8))
            add(k + '.bytes', 'bytes', np.frombuffer(b''.join(chunks), np.uint8))
        elif k in DEVICE_INT or k in DEVICE_FLOAT:
            add(k, 'array', _narrow([f[k] for f in features]))
    # two-pass layout: the header length fixes the first offset
    header = {'n': n, 'max_seq_len': max_seq_len, 'columns': cols}
    for c in cols:
        c['offset'], c['nbytes'] = 0, 0
    hlen = len(json.dumps(header).encode()) + 48 * len(cols) + 64      # room for the real offsets
    off = (16 + hlen + _ALIGN - 1) // _ALIGN * _ALIGN
    for c, b in zip(cols, blobs):
        c['offset'], c['nbytes'] = off, int(b.nbytes)
        off = (off + b.nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
    hjson = json.dumps(header).encode()
    assert len(hjson) <= hlen
    hjson = hjson + b' ' * (hlen - len(hjson))
    tmp = path + '.tmp'
    with open(tmp, 'wb') as f:
        f.write(MAGIC)
        f.write(np.uint64(hlen).tobytes())
        f.write(hjson)
        for c, b in zip(cols, blobs):
            f.seek(c['offset'])
            f.write(b.tobytes())
        f.truncate(off)
    os.replace(tmp, path)
    return header


class RecordFile(object):
    """Memory-mapped reader of one .nerrec file."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            if f.read(8) != MAGIC:
                raise ValueError('{}: not a .nerrec file'.format(path))
            hlen = int(np.frombuffer(f.read(8), np.uint64)[0])
            self.header = json.loads(f.read(hlen).decode())
        self.n, self.max_seq_len = self.header['n'], self.header['max_seq_len']
        self._mm = np.memmap(path, dtype=np.uint8, mode='r')
        self.cols, self._byteptr = {}, {}
        for c in self.header['columns']:
            raw = self._mm[c['offset']:c['offset'] + c['nbytes']]
            self.cols[c['name']] = (c['kind'], raw.view(np.dtype(c['dtype'])).reshape(c['shape']))

    def __len__(self):
        return self.n

    def names(self):
        return [k for k, (kind, _) in self.cols.items() if kind != 'bytes']

    def strings(self, name, rows):
        """[len(rows), L] python strings of a 'strings' column."""
        rowptr, lens, blob = self.cols[name][1], self.cols[name + '.len'][1], self.cols[name + '.bytes'][1]
        bptr = self._byteptr.get(name)
        if bptr is None:                      # byte offset of every stored entry, built once per column
            bptr = self._byteptr[name] = np.concatenate([[0], np.cumsum(lens, dtype=np.int64)])
        L, out = self.max_seq_len, []
        for r in rows:
            a, b = int(rowptr[r]), int(rowptr[r + 1])
            o = bptr[a:b + 1]
            raw, base = bytes(blob[o[0]:o[-1]]), int(o[0])
            row = [raw[int(o[i]) - base:int(o[i + 1]) - base].decode('utf-8') for i in range(b - a)]
            out.append(row + [PAD_STRING] * (L - len(row)))
        return out

    def batch(self, rows, pin_memory=False, with_strings=True):
        """rows: index array / slice -> the feature dict of dataset.py:21-37 (int32 / float32 tensors, string lists)."""
        if isinstance(rows, slice):
            rows = np.arange(*rows.indices(self.n))
        rows = np.asarray(rows, dtype=np.int64)
        out = {}
        for name, (kind, arr) in self.cols.items():
            if kind == 'array':
                a = arr[rows]
                t = torch.from_numpy(a.astype(np.float32 if name in DEVICE_FLOAT else np.int32))
                out[name] = t.pin_memory() if (pin_memory and torch.cuda.is_available()) else t
            elif kind == 'strings' and with_strings:
                out[name] = self.strings(name, rows)
        return out


def shuffle_window(n, buffer_size, rng):
    """Index order of tf.data's `shuffle(buffer_size)` over range(n): a buffer of `buffer_size` elements, each output
    drawn uniformly from it and replaced by the next input (dataset.py:47 uses buffer_size=64)."""
    out = np.empty(n, np.int64)
    buf = list(range(min(buffer_size, n)))
    nxt = len(buf)
    draws = rng.random(n)
    for i in range(n):
        j = int(draws[i] * len(buf))
        out[i] = buf[j]
        if nxt < n:
            buf[j] = nxt
            nxt += 1
        else:
            buf[j] = buf[-1]
            buf.pop()
    return out


class NerDataset(object):
    """reference dataset.py:12-71 over .nerrec files: same constructor, `params`, `build_input_fn(file_name, is_predict)`.

    `build_input_fn(...)()` returns an iterator of host feature batches (pinned): not is_predict ->
    shuffle(64).repeat(epoch_size).batch(batch_size) — batches run across epoch boundaries exactly as tf.data's do, the
    last one may be short —, is_predict -> one ordered pass."""

    def __init__(self, data_dir, batch_size, epoch_size, model_name, seed=1234):
        from .base_preprocess import extract_prefix_surfix
        self.surfix, self.prefix = extract_prefix_surfix(model_name)
        self.data_dir, self.batch_size, self.epoch_size, self.seed = data_dir, batch_size, epoch_size, seed
        self._params = None
        self.init_params()

    def file_path(self, file_name):
        return os.path.join(self.data_dir, '_'.join(filter(None, [self.prefix, file_name, self.surfix])) + '.nerrec')

    def init_params(self):
        with open(os.path.join(self.data_dir, '_'.join(filter(None, [self.prefix, self.surfix, 'data_params.pkl']))), 'rb') as f:
            self._params = pickle.load(f)
        self._params['step_per_epoch'] = int(self._params['n_sample'] / self.batch_size)
        self._params['num_train_steps'] = int(self.epoch_size * self._params['step_per_epoch'])

    @property
    def params(self):
        return self._params

    def build_input_fn(self, file_name, is_predict=0, pin_memory=True, with_strings=None):
        path = self.file_path(file_name)
        with_strings = bool(is_predict) if with_strings is None else with_strings

        def input_fn():
            rec = RecordFile(path)
            B = self.batch_size
            if is_predict:
                for s in range(0, rec.n, B):
                    yield rec.batch(slice(s, min(s + B, rec.n)), pin_memory, with_strings)
                return
            rng = np.random.default_rng(self.seed)
            carry = np.empty(0, np.int64)
            for _ in range(self.epoch_size):
                order = np.concatenate([carry, shuffle_window(rec.n, 64, rng)])
                full = len(order) // B * B
                for s in range(0, full, B):
                    yield rec.batch(order[s:s + B], pin_memory, with_strings)
                carry = order[full:]
            if len(carry):
                yield rec.batch(carry, pin_memory, with_strings)
        return input_fn


class MultiDataset(object):
    """reference dataset.py:73-141 over .nerrec files — the input pipe of the multi-task / adversarial plugins: one
    NerDataset per directory, batches mix the datasets sample by sample and carry `task_ids` (the index of the dataset a
    sentence came from).

    `build_input_fn(file_name)`: the datasets are shuffled (window 64) and interleaved one sample at a time
    (`choose_from_datasets` over `range(n).repeat()`; a dataset that runs out is skipped and the others continue until all
    are exhausted), the interleaved stream is repeated `epoch_size` times and cut into batches.  `build_predict_fn(data)`:
    one ordered pass over that dataset's `predict` split.  `params`: each dataset's params under its name, `task_list`,
    `step_per_epoch` (the largest of the datasets', as the reference takes it), `num_train_steps`, `max_seq_len`."""

    def __init__(self, root_dir, data_list, batch_size, epoch_size, model_name, seed=1234):
        self.batch_size, self.epoch_size, self.data_list, self.seed = batch_size, epoch_size, list(data_list), seed
        self.dataset_dict = OrderedDict((d, NerDataset(os.path.join(root_dir, d), batch_size, epoch_size, model_name, seed))
                                        for d in self.data_list)
        self._params = {}
        self.init_params()

    def init_params(self):
        for data, dataset in self.dataset_dict.items():
            self._params[data] = dataset.params
        self._params['step_per_epoch'] = int(max(p['step_per_epoch'] for p in self._params.values()))
        self._params['num_train_steps'] = int(self.epoch_size * self._params['step_per_epoch'])
        self._params['task_list'] = self.data_list
        self._params['max_seq_len'] = self._params[self.data_list[0]]['max_seq_len']

    @property
    def params(self):
        return self._params

    @staticmethod
    def _collate(parts, pin_memory):
        """list of (task, single-row feature dict) -> one batch dict with task_ids [B]."""
        out = {}
        for k in parts[0][1]:
            vals = [f[k] for _, f in parts]
            out[k] = torch.cat(vals, 0) if torch.is_tensor(vals[0]) else [x for v in vals for x in v]
        out['task_ids'] = torch.tensor([t for t, _ in parts], dtype=torch.int32)
        if pin_memory and torch.cuda.is_available():
            out = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in out.items()}
        return out

    def build_input_fn(self, file_name, is_predict=0, pin_memory=True, with_strings=False):
        """is_predict (used for the EVAL passes): one ordered, unshuffled pass over the interleaved stream."""
        def input_fn():
            recs = [RecordFile(ds.file_path(file_name)) for ds in self.dataset_dict.values()]
            rng = np.random.default_rng(self.seed)
            pending = []

            def flush():
                return self._collate([(t, recs[t].batch([i], False, with_strings)) for t, i in pending], pin_memory)

            for _ in range(1 if is_predict else self.epoch_size):
                orders = [np.arange(r.n) if is_predict else shuffle_window(r.n, 64, rng) for r in recs]
                pos = [0] * len(recs)
                while any(p < len(o) for p, o in zip(pos, orders)):
                    for t, order in enumerate(orders):                        # choice dataset = 0, 1, ..., 0, 1, ...
                        if pos[t] < len(order):
                            pending.append((t, int(order[pos[t]])))
                            pos[t] += 1
                            if len(pending) == self.batch_size:
                                yield flush()
                                pending = []
            if pending:
                yield flush()
        return input_fn

    def build_predict_fn(self, data, pin_memory=True):
        task = self.data_list.index(data)
        inner = self.dataset_dict[data].build_input_fn('predict', is_predict=True, pin_memory=False)

        def input_fn():
            for feats in inner():
                feats['task_ids'] = torch.full((feats['token_ids'].shape[0],), task, dtype=torch.int32)
                if pin_memory and torch.cuda.is_available():
                    feats = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in feats.items()}
                yield feats
        return input_fn
