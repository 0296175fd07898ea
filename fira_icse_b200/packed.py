"""Per-commit packed batches (SURVEY.md 8f rank 4): node rows = the REAL nodes of every commit instead of the
reference's fixed 210 / 160 / 280 padding (Dataset.py:80-94).

Row layout of the encoder's node buffer for a packed batch (segment-major, ragged):

    [ code rows of commit 0 | commit 1 | ... | pad to Rc ][ sub-token rows ... | pad to Rs ][ AST/edit rows ... | pad to Ra ]

`off[s][b]` is the first row of commit b inside segment s; padding rows carry id 0 and have no edges.  The adjacency
comes as a CSR in buffer order with global column ids, the decoder memory of commit b is the two row ranges
`ranges[b] = (first code row, code rows, first sub-token row, sub-token rows)` -- no `torch.cat`, no pack kernel --
and copy labels are renumbered to the commit's own memory rows (V + m, m < code rows + sub rows).  Everything a
padded batch computes on real rows is reproduced exactly: padding nodes are isolated in the graph and masked in
cross-attention and the copy softmax (SURVEY.md 9.3), so they never reach a real row or the loss.
"""
import numpy as np
import torch

from ._lib import host_call

SEGMENT_BUCKETS = (1024, 512, 512, 64)          # rounding of (code rows, sub rows, AST rows, memory rows per commit)
VOCAB_ROW_BUCKET = 128                          # rounding of the vocabulary-label and live target rows: one GEMM row tile


class PackedBatch:
    """Tensors of one packed batch (host or device) + its static dimensions."""

    FIELDS = ("code", "mark", "pos", "sub", "ast", "off", "ranges", "mem_mask", "tar", "label", "tar_mask",
              "rowptr", "col", "val")

    def __init__(self, B, Rc, Rs, Ra, S, T, nnz, chunks=4, Rv=None, Rt=None, **tensors):
        self.B, self.Rc, self.Rs, self.Ra, self.S, self.T, self.nnz = B, Rc, Rs, Ra, S, T, nnz
        # bound on the 128-key chunks cross-attention needs for any commit of the batch (3 on the whole shipped DataSet:
        # <= 200 code tokens, <= 102 sub-tokens); passed to the packed attention entry points, which do not use it
        self.chunks = int(chunks)
        # bound on the target rows whose label is a vocabulary word: the rows of the training step's vocabulary
        # projection (ops.HeadFn); None = every row
        self.Rv = B * T if Rv is None else int(Rv)
        # bound on the live target rows, the rows before each commit's last label (>= Rv): the rows of the training
        # step's decoder backward (ops.DecoderFn); None = every row
        self.Rt = B * T if Rt is None else int(Rt)
        for k in self.FIELDS:
            setattr(self, k, tensors[k])

    @property
    def shape_key(self):
        return (self.B, self.Rc, self.Rs, self.Ra, self.S, self.chunks, self.Rt, self.Rv)

    @property
    def rows(self):
        return self.Rc + self.Rs + self.Ra

    @property
    def mem_rows(self):
        return self.Rc + self.Rs

    def to(self, device, non_blocking=True):
        t = {k: getattr(self, k).to(device, non_blocking=non_blocking) for k in self.FIELDS}
        return PackedBatch(self.B, self.Rc, self.Rs, self.Ra, self.S, self.T, self.nnz, self.chunks, self.Rv, self.Rt, **t)

    def h2d_bytes(self):
        return sum(getattr(self, k).numel() * getattr(self, k).element_size() for k in self.FIELDS)


def _round_up(x, m):
    return max(m, -(-int(x) // m) * m)


class PackedTables:
    """The int32 / uint8 / int16 / float64 split arrays of a TransDataset (or synth.SynthDataset) in the form the
    native gather reads, shared by every packed batch built from that dataset."""

    ID_KEYS = ("sou", "tar", "mark", "ast_change", "tar_label", "sub_token")

    def __init__(self, dataset):
        d = dataset.d
        self.tab = {k: np.ascontiguousarray(d[k], dtype=np.int32) for k in self.ID_KEYS}
        self.deg = np.ascontiguousarray(d["deg"], dtype=np.uint8)
        self.col = np.ascontiguousarray(d["col"], dtype=np.int16)
        self.val = np.ascontiguousarray(d["val"], dtype=np.float64)
        self.edge_ptr = np.ascontiguousarray(d["edge_ptr"], dtype=np.int64)
        self.lens = (dataset.diff_len, dataset.sub_token_len, dataset.ast_change_len)
        self.msg_len = dataset.msg_len
        self.n = len(self.tab["sou"])

    def dims(self, index):
        """-> (code rows, sub rows, AST rows, max memory rows of one commit, nnz, attention key chunks) of `index`"""
        index = np.ascontiguousarray(index, dtype=np.int64)
        t = self.tab
        out = np.zeros(6, np.int32)
        host_call("fira_host_packed_dims", t["sou"].ctypes.data, t["sub_token"].ctypes.data, t["ast_change"].ctypes.data,
                  self.deg.ctypes.data, index.ctypes.data, len(index), *self.lens, out.ctypes.data)
        return tuple(int(x) for x in out)

    def vocab_rows(self, index, vocab_size):
        """-> target rows of `index` whose shifted label is a vocabulary word (0 < label < V; fira_host_gather_packed
        renumbers copy labels only, so the count is the same before and after the gather)"""
        lab = self.tab["tar_label"][np.asarray(index, dtype=np.int64), 1:]
        return int(np.count_nonzero((lab > 0) & (lab < vocab_size)))

    def live_rows(self, index):
        """-> target rows of `index` before each commit's last non-zero shifted label (the count of fira_target_rows)"""
        lab = self.tab["tar_label"][np.asarray(index, dtype=np.int64), 1:] != 0
        last = lab.shape[1] - np.argmax(lab[:, ::-1], axis=1)
        return int(np.where(lab.any(axis=1), last, 0).sum())


class PackedSlot:
    """Staging buffers (pinned when CUDA is present) sized for the largest packed batch of `B` commits."""

    def __init__(self, B, lens, msg_len, edge_cap, pin):
        n0, n1, n2 = lens

        def buf(n, dt):
            t = torch.empty(n, dtype=dt)
            return t.pin_memory() if pin else t
        i32, u8 = torch.int32, torch.uint8
        self.cap = (_round_up(B * n0, SEGMENT_BUCKETS[0]), _round_up(B * n1, SEGMENT_BUCKETS[1]),
                    _round_up(B * n2, SEGMENT_BUCKETS[2]), _round_up(n0 + n1, SEGMENT_BUCKETS[3]))
        Rc, Rs, Ra, S = self.cap
        self.code, self.mark, self.pos = buf(Rc, i32), buf(Rc, i32), buf(Rc, i32)
        self.sub, self.ast = buf(Rs, i32), buf(Ra, i32)
        self.off, self.ranges = buf(3 * (B + 1), i32), buf(4 * B, i32)
        self.mem_mask = buf(B * S, u8)
        self.tar, self.label, self.tar_mask = buf(B * msg_len, i32), buf(B * msg_len, i32), buf(B * msg_len, u8)
        self.rowptr = buf(Rc + Rs + Ra + 1, i32)
        self.col, self.val = buf(edge_cap, i32), buf(edge_cap, torch.float32)
        self.edge_cap = edge_cap
        self.event = None
        self.batch = None


def gather_packed(tables, index, vocab_size, slot, pad_dims=None, buckets=SEGMENT_BUCKETS):
    """One packed batch of commits `index` written into `slot` (views of the slot are returned as a PackedBatch).
    pad_dims: (Rc, Rs, Ra, S[, Rv[, Rt]]) to use (>= the batch's needs, packed_needs); default = the needs rounded up
    to `buckets`.  Rv and Rt are capped at the batch's target rows; an Rt not given is the need, at least Rv."""
    index = np.ascontiguousarray(index, dtype=np.int64)
    b = len(index)
    need = tables.dims(index)
    if pad_dims is None:
        pad_dims = packed_needs(tables, index, vocab_size, buckets)
    elif len(pad_dims) < 6:
        need_all = packed_needs(tables, index, vocab_size, buckets)
        pad_dims = tuple(pad_dims) + need_all[len(pad_dims):]
        pad_dims = pad_dims[:5] + (max(pad_dims[4], pad_dims[5]),)
    Rc, Rs, Ra, S, Rv, Rt = (int(x) for x in pad_dims)
    if Rc > slot.cap[0] or Rs > slot.cap[1] or Ra > slot.cap[2] or S > slot.cap[3]:
        raise ValueError(f"packed batch {pad_dims} exceeds the staging capacity {slot.cap}")
    if Rv < tables.vocab_rows(index, vocab_size):
        raise ValueError(f"packed batch: Rv = {Rv} is below its vocabulary-label rows")
    if Rt < max(Rv, tables.live_rows(index)):
        raise ValueError(f"packed batch: Rt = {Rt} is below its live target rows or Rv = {Rv}")
    t = tables.tab
    pd = np.asarray((Rc, Rs, Ra, S), np.int32)
    nnz = np.zeros(1, np.int32)
    host_call("fira_host_gather_packed", t["sou"].ctypes.data, t["tar"].ctypes.data, t["mark"].ctypes.data,
              t["ast_change"].ctypes.data, t["tar_label"].ctypes.data, t["sub_token"].ctypes.data,
              tables.deg.ctypes.data, tables.col.ctypes.data, tables.val.ctypes.data, tables.edge_ptr.ctypes.data,
              index.ctypes.data, b, *tables.lens, tables.msg_len, int(vocab_size), pd.ctypes.data,
              slot.code.data_ptr(), slot.mark.data_ptr(), slot.pos.data_ptr(), slot.sub.data_ptr(), slot.ast.data_ptr(),
              slot.off.data_ptr(), slot.ranges.data_ptr(), slot.mem_mask.data_ptr(), slot.tar.data_ptr(),
              slot.label.data_ptr(), slot.tar_mask.data_ptr(), slot.rowptr.data_ptr(), slot.col.data_ptr(),
              slot.val.data_ptr(), slot.edge_cap, nnz.ctypes.data)
    e, T = int(nnz[0]), tables.msg_len
    slot.batch = PackedBatch(
        b, Rc, Rs, Ra, S, T, e, max(3, need[5]), min(Rv, b * T), min(Rt, b * T),
        code=slot.code[:Rc], mark=slot.mark[:Rc], pos=slot.pos[:Rc], sub=slot.sub[:Rs], ast=slot.ast[:Ra],
        off=slot.off[:3 * (b + 1)].view(3, b + 1), ranges=slot.ranges[:4 * b].view(b, 4),
        mem_mask=slot.mem_mask[:b * S].view(b, S), tar=slot.tar[:b * T].view(b, T), label=slot.label[:b * T].view(b, T),
        tar_mask=slot.tar_mask[:b * T].view(b, T), rowptr=slot.rowptr[:Rc + Rs + Ra + 1], col=slot.col[:e],
        val=slot.val[:e])
    return slot.batch


def packed_needs(tables, index, vocab_size, buckets=SEGMENT_BUCKETS):
    """-> (Rc, Rs, Ra, S, Rv, Rt) of commits `index`: the rows each segment needs rounded up to `buckets`, the
    vocabulary-label target rows and the live target rows rounded up to VOCAB_ROW_BUCKET (Rt >= Rv), capped at the
    batch's target rows"""
    need = tables.dims(index)
    cap = len(index) * tables.msg_len
    Rv = min(_round_up(tables.vocab_rows(index, vocab_size), VOCAB_ROW_BUCKET), cap)
    Rt = min(max(_round_up(tables.live_rows(index), VOCAB_ROW_BUCKET), Rv), cap)
    return tuple(_round_up(need[i], buckets[i]) for i in range(4)) + (Rv, Rt)


def pack_from_dataset(dataset, index, vocab_size, pin=False, pad_dims=None, buckets=SEGMENT_BUCKETS):
    """Convenience for tests / tools: one packed batch with its own staging buffers."""
    tables = dataset if isinstance(dataset, PackedTables) else PackedTables(dataset)
    per_commit = int(np.diff(tables.edge_ptr).max()) if len(tables.edge_ptr) > 1 else 0
    slot = PackedSlot(len(index), tables.lens, tables.msg_len, max(1, per_commit * len(index)), pin)
    return gather_packed(tables, index, vocab_size, slot, pad_dims=pad_dims, buckets=buckets)
