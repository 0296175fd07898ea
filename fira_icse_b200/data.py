"""`Dataset.py` surface of the reference (TransDataset) with a packed on-disk/in-memory format.

Same inputs (CWD-relative DataSet/*.json, VOCAB_UPPER_CASE, all_index), same id conversion,
padding, dual-copy labels and adjacency definition as the reference (Dataset.py:96-294,346-357);
what changes is the representation handed to the model:

  reference: per item a dense float64 650x650 `toarray()` (3.38 MB/commit through collate + PCIe)
  here     : per item the CSR pieces (row degrees uint8[650], col int16[nnz], val fp32[nnz], ~6 KB);
             `collate_packed` concatenates them into one batch CSR (pinned host tensors) that
             PackedEdges.from_host ships with three async H2D copies.

`TransDataset[i]` still returns the reference's 8-element list (dense adjacency on request) so the
reference's own DataLoader/collate keeps working.
"""
import json
import os
import random

import numpy as np
import torch
from torch.utils.data import Dataset

from ._lib import host_call

num_train, num_valid, num_test = 75000, 8000, 7661          # Dataset.py:10-12
lemmatization = {"added": "add", "fixed": "fix", "removed": "remove",
                 "adding": "add", "fixing": "fix", "removing": "remove"}
RAW_FILES = ["difftoken", "diffatt", "diffmark", "msg", "variable", "change", "ast",
             "edge_change_code", "edge_change_ast", "edge_ast_code", "edge_ast"]


def _lower(tok, upper):
    return tok if tok in upper else tok.lower()


def _to_ids(tokens, vocab, upper):
    out = []
    for t in tokens:
        t = _lower(t, upper)
        out.append(vocab[t] if t in vocab else vocab["<unkm>"])     # lazy like Dataset.py:75-78
    return out


def _fit(seq, n):
    return (list(seq) + [0] * n)[:n]


def _pairs(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.int32).reshape(-1, 2))


def build_adjacency(change_code, change_ast, ast_code, ast_ast, code_sub, n_diff, n_ast, diff_len=210, sub_len=160,
                    ast_change_len=280):
    """Commit graph of Dataset.py:220-294,346-357 through the native builder (fira_host_build_adjacency):
    relation pair lists as stored in DataSet/edge_*.json -> (deg int32[n_nodes], col int32[nnz], val f64[nnz])
    in CSR order; undirected, de-duplicated, self loop on every node, value 1/sqrt(deg_r)/sqrt(deg_c)."""
    rel = [_pairs(r) for r in (change_code, change_ast, ast_code, ast_ast, code_sub)]
    n_nodes = diff_len + sub_len + ast_change_len
    cap = 2 * (sum(len(r) for r in rel) + n_diff + 1) + n_nodes
    deg = np.empty(n_nodes, np.int32)
    col = np.empty(cap, np.int32)
    val = np.empty(cap, np.float64)
    nnz = np.zeros(1, np.int32)
    args = []
    for r in rel:
        args += [r.ctypes.data, len(r)]
    host_call("fira_host_build_adjacency", *args, int(n_diff), int(n_ast), diff_len, sub_len, ast_change_len,
              deg.ctypes.data, col.ctypes.data, val.ctypes.data, cap, nnz.ctypes.data)
    return deg, col[:nnz[0]].copy(), val[:nnz[0]].copy()


def _diff_words(raw, i, upper):
    var_map = raw["variable"][i]
    return [_lower(var_map.get(t, t), upper) for t in raw["difftoken"][i]]


def _msg_words(words, var_map, upper):
    """message words as the labels see them: variable map, case, lemmatisation"""
    return [lemmatization.get(w, w) for w in (_lower(var_map.get(t, t), upper) for t in words)]


def _sub_tokens(diff, atts):
    """sub-token nodes, shared by repeated identifiers (first occurrence defines them) -> (sub-tokens, code-sub pairs)"""
    sub_tokens, owner, code_sub = [], {}, []
    for j, att in enumerate(atts):
        if att:
            if diff[j] not in owner:
                owner[diff[j]] = range(len(sub_tokens), len(sub_tokens) + len(att))
                sub_tokens.extend(att)
            code_sub.extend((j, k) for k in owner[diff[j]])
    return sub_tokens, code_sub


def _dual_copy_labels(msg, msg_ids, diff, sub_tokens, V, diff_len):
    """dual-copy labels: position in the diff wins over position among the sub-tokens, then the vocabulary id"""
    first_in_diff, first_in_sub = {}, {}
    for j, t in enumerate(diff):
        first_in_diff.setdefault(t, j)
    for k, t in enumerate(sub_tokens):
        first_in_sub.setdefault(t, k)
    label = []
    for w, wid in zip(msg, msg_ids):
        if w in first_in_diff:
            label.append(first_in_diff[w] + V + 1)
        elif w in first_in_sub:
            label.append(first_in_sub[w] + V + diff_len)
        else:
            label.append(wid)
    return label


def prefix_labels(raw, i, words, vocab, upper, diff_len=210):
    """Words a user typed as the start of commit i's message -> their labels in the tar_label encoding (without
    <start>), for the decoders' `prefix`: build_commit's normalisation and dual-copy label rule, so the labels of a
    message's first n words are tar_label[1:1 + n] of that message."""
    var_map = raw["variable"][i]
    diff = _diff_words(raw, i, upper)
    sub_tokens, _ = _sub_tokens(diff, raw["diffatt"][i])
    msg = _msg_words(words, var_map, upper)
    return _dual_copy_labels(msg, _to_ids(msg, vocab, upper), diff, sub_tokens, len(vocab), diff_len)


def constraint_words(raw, i, phrases, vocab, upper):
    """Words a user requires in commit i's message -> their vocabulary ids, for nbest's `constraints`: phrases is a list
    of phrases, each a string of words separated by spaces or a list of words, normalised as build_commit normalises
    message words (variable map, case, lemmatisation) -> a list of id lists.  ValueError for a word that maps to
    <unkm>: it has no id a hypothesis could contain."""
    var_map = raw["variable"][i]
    out = []
    for ph in phrases:
        words = ph.split() if isinstance(ph, str) else list(ph)
        ids = _to_ids(_msg_words(words, var_map, upper), vocab, upper)
        for w, wid in zip(words, ids):
            if wid == vocab["<unkm>"]:
                raise ValueError(f"constraint word {w!r} of commit {i} is not in the vocabulary (<unkm>)")
        out.append(ids)
    return out


def build_commit(raw, i, vocab, ast_vocab, upper, diff_len=210, msg_len=30, att_len=25, ast_change_len=280,
                 sub_len=160):
    """One commit -> padded id arrays + CSR pieces of its normalised adjacency.

    Node ids: code token j -> j+1 (0 = <start>), sub-token k -> 210+k, AST node a -> 370+a,
    edit node c -> 370+len(ast)+c.  Edges: edit-code, edit-AST, AST-code, AST-AST, code-sub-token,
    sequential code chain; undirected, de-duplicated; self loop on all 650 nodes;
    value 1/sqrt(deg_row)/sqrt(deg_col) in float64."""
    var_map = raw["variable"][i]
    diff = _diff_words(raw, i, upper)
    msg = _msg_words(raw["msg"][i], var_map, upper)
    atts = raw["diffatt"][i]
    V = len(vocab)
    n_ast = len(raw["ast"][i])

    sou = _fit([vocab["<start>"]] + _to_ids(diff, vocab, upper) + [vocab["<eos>"]], diff_len)
    msg_ids = _to_ids(msg, vocab, upper)
    tar = _fit([vocab["<start>"]] + msg_ids + [vocab["<eos>"]], msg_len)
    mark = _fit([2] + list(raw["diffmark"][i]) + [2], diff_len)
    ast_change = _fit(_to_ids(list(raw["ast"][i]) + list(raw["change"][i]), ast_vocab, upper), ast_change_len)

    sub_tokens, code_sub = _sub_tokens(diff, atts)
    sub_token = _fit(_to_ids(sub_tokens, vocab, upper), sub_len)

    label = _dual_copy_labels(msg, msg_ids, diff, sub_tokens, V, diff_len)
    tar_label = _fit([vocab["<start>"]] + label + [vocab["<eos>"]], msg_len)

    deg_r, col, val = build_adjacency(raw["edge_change_code"][i], raw["edge_change_ast"][i], raw["edge_ast_code"][i],
                                      raw["edge_ast"][i], code_sub, len(diff), n_ast, diff_len, sub_len, ast_change_len)
    if deg_r.max() > 255:
        raise ValueError("a node has more than 255 neighbours: the packed degree table is uint8")
    attr_pos = [j + 1 for j, att in enumerate(atts) if att]           # row of the padded [210,25] attr matrix
    attr_ids = [_fit(_to_ids(atts[j - 1], vocab, upper), att_len) for j in attr_pos]
    return dict(sou=sou, tar=tar, mark=mark, ast_change=ast_change, tar_label=tar_label, sub_token=sub_token,
                deg=deg_r.astype(np.uint8), col=col.astype(np.int16), val=val,
                attr_pos=[p for p in attr_pos if p < diff_len], attr_ids=attr_ids[:sum(p < diff_len for p in attr_pos)])


class TransDataset(Dataset):
    """TransDataset(args, 'train'|'valid'|'test'[, root='.'])  (Dataset.py:17-68)."""

    ID_KEYS = ("sou", "tar", "mark", "ast_change", "tar_label", "sub_token")

    def __init__(self, args, data_name, root=".", dense_edges=False, limit=None):
        super().__init__()
        self.data_name = data_name
        self.diff_len, self.msg_len, self.att_len = args.sou_len, args.tar_len, args.att_len
        self.ast_change_len, self.sub_token_len = args.ast_change_len, args.sub_token_len
        self.graph_len = self.diff_len + self.sub_token_len + self.ast_change_len
        self.dense_edges = dense_edges
        self.root = root
        # a truncated build (limit=N) gets its own cache name: a later full run must not pick it up
        self._tag = f"_limit{int(limit)}" if limit else ""
        cache = os.path.join(root, f"processed_b200_{data_name}{self._tag}.npz")
        if not os.path.exists(cache):
            self._process_all(limit)
        z = np.load(cache)
        self.d = {k: z[k] for k in z.files}
        print("Loaded data!")

    # ------------------------------------------------------------------ one-off preprocessing
    def _process_all(self, limit=None):
        j = lambda n: json.load(open(os.path.join(self.root, "DataSet", n + ".json")))
        raw = {n: j(n) for n in RAW_FILES}
        n_all = len(raw["difftoken"])
        assert all(len(raw[n]) == n_all for n in RAW_FILES)
        vocab, ast_vocab = j("word_vocab"), j("ast_change_vocab")
        upper = set(json.load(open(os.path.join(self.root, "VOCAB_UPPER_CASE"))))
        idx_path = os.path.join(self.root, "all_index")
        if os.path.exists(idx_path):
            all_index = json.load(open(idx_path))
        else:                                      # Dataset.py:306-313 under seed_everything(0)
            index = list(range(n_all))
            random.Random(0).shuffle(index)
            nt, nv = min(num_train, int(n_all * 0.83)), min(num_valid, int(n_all * 0.09))
            all_index = {"train": index[:nt], "valid": index[nt:nt + nv], "test": index[nt + nv:]}
            json.dump(all_index, open(idx_path, "w"))
        for split, order in all_index.items():
            if limit:
                order = order[:limit]
            cols = {k: [] for k in self.ID_KEYS}
            deg, col, val, eptr = [], [], [], [0]
            apos, aids, aptr = [], [], [0]
            for i in order:
                c = build_commit(raw, i, vocab, ast_vocab, upper, self.diff_len, self.msg_len, self.att_len,
                                 self.ast_change_len, self.sub_token_len)
                for k in self.ID_KEYS:
                    cols[k].append(c[k])
                deg.append(c["deg"]); col.append(c["col"]); val.append(c["val"]); eptr.append(eptr[-1] + len(c["col"]))
                apos += c["attr_pos"]; aids += c["attr_ids"]; aptr.append(aptr[-1] + len(c["attr_pos"]))
            np.savez(os.path.join(self.root, f"processed_b200_{split}{self._tag}.npz"),
                     **{k: np.array(v, np.int32).reshape(len(order), -1) for k, v in cols.items()},
                     deg=np.array(deg, np.uint8).reshape(len(order), self.graph_len),
                     col=np.concatenate(col) if col else np.zeros(0, np.int16),
                     val=np.concatenate(val) if val else np.zeros(0, np.float64), edge_ptr=np.array(eptr, np.int64),
                     attr_pos=np.array(apos, np.int16), attr_ids=np.array(aids, np.int32).reshape(-1, self.att_len),
                     attr_ptr=np.array(aptr, np.int64), index=np.array(order, np.int64))

    # ------------------------------------------------------------------ access
    def __len__(self):
        return len(self.d["sou"])

    def csr_pieces(self, i):
        lo, hi = self.d["edge_ptr"][i], self.d["edge_ptr"][i + 1]
        return self.d["deg"][i], self.d["col"][lo:hi], self.d["val"][lo:hi]

    def attr(self, i):
        out = np.zeros((self.diff_len, self.att_len), np.int64)
        lo, hi = self.d["attr_ptr"][i], self.d["attr_ptr"][i + 1]
        out[self.d["attr_pos"][lo:hi]] = self.d["attr_ids"][lo:hi]
        return out

    def dense_edge(self, i):
        deg, col, val = self.csr_pieces(i)
        a = np.zeros((self.graph_len, self.graph_len), np.float64)
        a[np.repeat(np.arange(self.graph_len), deg), col] = val
        return a

    def __getitem__(self, i):
        d = self.d
        edge = self.dense_edge(i) if self.dense_edges else self.csr_pieces(i)
        return [d["sou"][i].astype(np.int64), d["tar"][i].astype(np.int64), self.attr(i), d["mark"][i].astype(np.int64),
                d["ast_change"][i].astype(np.int64), edge, d["tar_label"][i].astype(np.int64),
                d["sub_token"][i].astype(np.int64)]


def collate_packed(items, pin=False):
    """list of TransDataset items (csr pieces) -> the 8-element batch with item 5 = host CSR triple
    (rowptr int32 [B*650+1], col int32, val fp32).  `attr` is dropped (None): the model ignores it."""
    def stack(k):
        return torch.from_numpy(np.stack([it[k] for it in items]))
    deg = np.concatenate([it[5][0] for it in items]).astype(np.int64)
    rowptr = torch.from_numpy(np.concatenate((np.zeros(1, np.int64), np.cumsum(deg))).astype(np.int32))
    col = torch.from_numpy(np.concatenate([it[5][1] for it in items]).astype(np.int32))
    val = torch.from_numpy(np.concatenate([it[5][2] for it in items]).astype(np.float32))
    out = [stack(0), stack(1), None, stack(3), stack(4), (rowptr, col, val), stack(6), stack(7)]
    if pin:
        out = [tuple(x.pin_memory() for x in o) if isinstance(o, tuple) else (o.pin_memory() if o is not None else None)
               for o in out]
    return out


def batch_to_device(batch, device, n_nodes=650):
    """collate_packed output -> model inputs on `device` (async copies from pinned memory)."""
    from .graph import PackedEdges
    out = []
    for j, o in enumerate(batch):
        if j == 5:
            B = batch[0].shape[0]
            out.append(PackedEdges.from_host(*o, B, n_nodes, device))
        else:
            out.append(o.to(device, non_blocking=True) if o is not None else None)
    return out


def trim_batch_host(batch, vocab_size, multiple=8, full=(210, 160, 280)):
    """Drop the padding the whole batch shares (var-len packing, SURVEY.md section 8f rank 4, loader side).

    batch: collate_packed-style list [sou, tar, attr, mark, ast_change, (rowptr, col, val), tar_label, sub_token]
    (host tensors, node lengths `full`).  Code / sub-token / AST+edit segments are cut to the longest
    commit of the batch (rounded up to `multiple`); the adjacency rows of the removed nodes -- isolated
    self-loop rows by construction (Dataset.py:271-275) -- are dropped, column ids and sub-token copy
    labels are renumbered.  Real rows, loss and gradients are unchanged; the model takes the shorter
    tensors as they are (all shapes are read from the inputs)."""
    sou, tar, attr, mark, ast_change, (rowptr, col, val), tar_label, sub_token = batch
    n0, n1, n2 = full
    B = sou.shape[0]

    def cap(t, n):
        nz = (t != 0).any(0).nonzero()
        used = int(nz.max()) + 1 if nz.numel() else 0            # position after the last non-padding id
        return min(n, max(multiple, -(-used // multiple) * multiple))
    c0, c1, c2 = cap(sou, n0), cap(sub_token, n1), cap(ast_change, n2)
    N, Nt = n0 + n1 + n2, c0 + c1 + c2
    keep = np.zeros(N, bool)
    keep[:c0] = True; keep[n0:n0 + c1] = True; keep[n0 + n1:n0 + n1 + c2] = True
    remap = np.full(N, -1, np.int64)
    remap[keep] = np.arange(Nt)
    rp = rowptr.numpy().astype(np.int64)
    deg = np.diff(rp).reshape(B, N)
    row_keep = np.broadcast_to(keep, (B, N)).reshape(-1)
    entry_keep = np.repeat(row_keep, deg.reshape(-1))
    new_col = remap[col.numpy()[entry_keep]]
    assert (new_col >= 0).all(), "a kept node has a neighbour inside the trimmed padding: adjacency is not padding-isolated"
    new_rowptr = np.concatenate((np.zeros(1, np.int64), np.cumsum(deg[:, keep].reshape(-1))))
    label = tar_label.clone()
    sub_copy = label >= vocab_size + n0
    label[sub_copy] -= (n0 - c0)
    out = [sou[:, :c0].contiguous(), tar, attr, mark[:, :c0].contiguous(), ast_change[:, :c2].contiguous(),
           (torch.from_numpy(new_rowptr.astype(np.int32)), torch.from_numpy(new_col.astype(np.int32)),
            torch.from_numpy(val.numpy()[entry_keep])), label, sub_token[:, :c1].contiguous()]
    return out


class _Slot:
    """One set of staging buffers (pinned when CUDA is present) sized for an untrimmed batch."""

    def __init__(self, B, lens, msg_len, edge_cap, pin):
        n0, n1, n2 = lens

        def buf(n, dt):
            t = torch.empty(n, dtype=dt)
            return t.pin_memory() if pin else t
        self.sou, self.mark = buf(B * n0, torch.int64), buf(B * n0, torch.int64)
        self.sub_token, self.ast_change = buf(B * n1, torch.int64), buf(B * n2, torch.int64)
        self.tar, self.tar_label = buf(B * msg_len, torch.int64), buf(B * msg_len, torch.int64)
        self.rowptr = buf(B * (n0 + n1 + n2) + 1, torch.int32)
        self.col, self.val = buf(edge_cap, torch.int32), buf(edge_cap, torch.float32)
        self.event = None
        self.batch = None


class PackedBatchLoader:
    """Native loader for a TransDataset: every batch is gathered, collated, padding-trimmed and CSR-packed by ONE
    call of fira_host_gather_batch (C++) into pinned staging buffers, on a background thread, `prefetch` batches
    ahead of the consumer.  Replaces DataLoader(dataset, collate_fn=...) + trim_batch_host.

    Yields the reference's 8-slot batch [sou, tar, None, mark, ast_change, (rowptr, col, val), tar_label,
    sub_token] as HOST tensors that are views of a staging slot: the consumer must enqueue its host->device
    copies (GraphedTrainStep.step / batch_to_device) before asking for the next batch -- the slot is recycled
    only after a CUDA event recorded at that moment has completed.

    multiples: rounding of the trimmed (code, sub-token, AST) segment lengths; None = no trimming.
    max_shapes: upper bound on the number of distinct batch shapes ever emitted (each shape is one captured
    CUDA graph downstream); once reached, a batch is padded up to the smallest already-emitted shape that
    holds it (the full 210/160/280 if none does).
    bucket: 0 (default) keeps the reference's batching -- consecutive slices of one uniform shuffle.  bucket = K > 1
    is an OPT-IN departure from it: the shuffled order is cut into windows of K batches, each window is sorted by
    commit size (real code + sub-token + AST nodes) before it is sliced, and the window's batches are emitted in
    random order.  Batches then hold commits of similar size, so trimming removes far more padding; every commit
    is still visited exactly once per epoch, but batch composition is no longer independent of commit size."""

    def __init__(self, dataset, batch_size, vocab_size, shuffle=False, indices=None, multiples=(8, 8, 8),
                 max_shapes=None, drop_last=False, prefetch=2, pin=None, bucket=0, packed=False, row_buckets=None):
        self.ds, self.B, self.V = dataset, int(batch_size), int(vocab_size)
        self.shuffle, self.drop_last = shuffle, drop_last
        self.bucket = int(bucket)
        self.indices = np.arange(len(dataset), dtype=np.int64) if indices is None else np.asarray(indices, np.int64)
        if len(self.indices) and (self.indices.min() < 0 or self.indices.max() >= len(dataset)):
            raise IndexError(f"PackedBatchLoader: indices must lie in [0, {len(dataset)}) "
                             f"(got {int(self.indices.min())}..{int(self.indices.max())}); the native gather does not "
                             "bounds-check")
        self.multiples = (0, 0, 0) if multiples is None else tuple(int(m) for m in multiples)
        self.max_shapes = max_shapes
        self.dims_used = {}            # every batch shape emitted (packed: Rc, Rs, Ra, S, Rv, Rt) -> batches
        self.lens = (dataset.diff_len, dataset.sub_token_len, dataset.ast_change_len)
        self.msg_len = dataset.msg_len
        d = dataset.d
        self.tab = {k: np.ascontiguousarray(d[k], dtype=np.int32) for k in TransDataset.ID_KEYS}
        self.deg = np.ascontiguousarray(d["deg"], dtype=np.uint8)
        self.col = np.ascontiguousarray(d["col"], dtype=np.int16)
        self.val = np.ascontiguousarray(d["val"], dtype=np.float64)
        self.edge_ptr = np.ascontiguousarray(d["edge_ptr"], dtype=np.int64)
        self.size = sum((self.tab[k] != 0).sum(1) for k in ("sou", "sub_token", "ast_change"))   # real nodes per commit
        per_commit = int(np.diff(self.edge_ptr).max()) if len(self.edge_ptr) > 1 else 0
        self.edge_cap = max(1, per_commit * self.B)
        self.pin = torch.cuda.is_available() if pin is None else pin
        self.n_slots = max(2, int(prefetch) + 1)
        # packed=True: per-commit packed batches (packed.PackedBatch, SURVEY.md 8f rank 4) instead of batch-trimmed padded
        # ones; row_buckets = rounding of (code rows, sub-token rows, AST rows, memory rows of one commit); the
        # vocabulary-label and live target rows round to packed.VOCAB_ROW_BUCKET, and max_shapes bounds the shapes with them
        self.packed = bool(packed)
        if self.packed:
            from . import packed as P
            self.tables = P.PackedTables(dataset)
            self.row_buckets = tuple(row_buckets) if row_buckets else P.SEGMENT_BUCKETS
            self.slots = [P.PackedSlot(self.B, self.lens, self.msg_len, self.edge_cap, self.pin)
                          for _ in range(self.n_slots)]
        else:
            self.slots = [_Slot(self.B, self.lens, self.msg_len, self.edge_cap, self.pin) for _ in range(self.n_slots)]

    def __len__(self):
        n = len(self.indices)
        return n // self.B if self.drop_last else -(-n // self.B)

    # ------------------------------------------------------------------ shape policy
    @property
    def shapes(self):
        """batches per emitted (code, sub-token, AST) lengths, or packed (Rc, Rs, Ra, S, Rv) rows"""
        out = {}
        for k, n in self.dims_used.items():
            out[k[:5]] = out.get(k[:5], 0) + n
        return out

    def _choose_dims(self, need):
        need = tuple(int(x) for x in need)
        used = self.dims_used
        if need in used or self.max_shapes is None or len(used) < self.max_shapes:
            used[need] = used.get(need, 0) + 1
            return need
        fits = [s for s in used if all(a >= b for a, b in zip(s, need))]
        if self.packed and not fits:                     # nothing emitted so far holds it: a new shape after all
            used[need] = 1
            return need
        best = min(fits, key=sum) if fits else self.lens
        used[best] = used.get(best, 0) + 1
        return best

    # ------------------------------------------------------------------ one batch
    def gather(self, index, slot=None):
        """index: int64 dataset positions -> batch (views of `slot`)."""
        slot = self.slots[0] if slot is None else slot
        index = np.ascontiguousarray(index, dtype=np.int64)
        if self.packed:
            from . import packed as P
            want = P.packed_needs(self.tables, index, self.V, self.row_buckets)
            return P.gather_packed(self.tables, index, self.V, slot, pad_dims=self._choose_dims(want))
        b = len(index)
        n0, n1, n2 = self.lens
        t = self.tab
        dims = np.zeros(3, np.int32)
        host_call("fira_host_batch_dims", t["sou"].ctypes.data, t["sub_token"].ctypes.data,
                  t["ast_change"].ctypes.data, index.ctypes.data, b, n0, n1, n2, *self.multiples, dims.ctypes.data)
        dims = np.asarray(self._choose_dims(dims), np.int32)
        nnz = np.zeros(1, np.int32)
        host_call("fira_host_gather_batch", t["sou"].ctypes.data, t["tar"].ctypes.data, t["mark"].ctypes.data,
                  t["ast_change"].ctypes.data, t["tar_label"].ctypes.data, t["sub_token"].ctypes.data,
                  self.deg.ctypes.data, self.col.ctypes.data, self.val.ctypes.data, self.edge_ptr.ctypes.data,
                  index.ctypes.data, b, n0, n1, n2, self.msg_len, self.V, dims.ctypes.data,
                  slot.sou.data_ptr(), slot.tar.data_ptr(), slot.mark.data_ptr(), slot.ast_change.data_ptr(),
                  slot.tar_label.data_ptr(), slot.sub_token.data_ptr(), slot.rowptr.data_ptr(), slot.col.data_ptr(),
                  slot.val.data_ptr(), self.edge_cap, nnz.ctypes.data)
        c0, c1, c2 = (int(x) for x in dims)
        e = int(nnz[0])
        slot.batch = [slot.sou[:b * c0].view(b, c0), slot.tar[:b * self.msg_len].view(b, self.msg_len), None,
                      slot.mark[:b * c0].view(b, c0), slot.ast_change[:b * c2].view(b, c2),
                      (slot.rowptr[:b * (c0 + c1 + c2) + 1], slot.col[:e], slot.val[:e]),
                      slot.tar_label[:b * self.msg_len].view(b, self.msg_len), slot.sub_token[:b * c1].view(b, c1)]
        return slot.batch

    # ------------------------------------------------------------------ iteration
    def epoch_batches(self):
        """Index arrays of one epoch's batches (draws from torch's global generator when shuffling)."""
        order = self.indices
        if self.shuffle:
            order = order[torch.randperm(len(order)).numpy()]        # torch's global generator, like DataLoader
        if self.bucket > 1:
            span = self.bucket * self.B
            chunks = []
            for lo in range(0, len(order), span):
                win = order[lo:lo + span]
                win = win[np.argsort(self.size[win], kind="stable")]
                part = [win[i:i + self.B] for i in range(0, len(win), self.B)]
                if self.shuffle and len(part) > 1:
                    part = [part[j] for j in torch.randperm(len(part)).tolist()]
                chunks += part
            if self.drop_last:
                chunks = [c for c in chunks if len(c) == self.B]
            else:                                                   # at most one short batch per window: keep them last
                chunks = [c for c in chunks if len(c) == self.B] + [c for c in chunks if len(c) < self.B]
            return chunks
        chunks = [order[i:i + self.B] for i in range(0, len(order), self.B)]
        if self.drop_last and chunks and len(chunks[-1]) < self.B:
            chunks.pop()
        return chunks

    def __iter__(self):
        import queue
        import threading
        chunks = self.epoch_batches()
        free_q, full_q = queue.Queue(), queue.Queue()
        # slot events survive from one epoch to the next: the copies of the previous epoch's last batches may still be
        # queued behind graph replays when the next epoch's producer starts refilling the staging slots
        for s in self.slots:
            free_q.put(s)
        stop = threading.Event()

        def produce():
            try:
                for ch in chunks:
                    s = free_q.get()
                    if stop.is_set():
                        return
                    if s.event is not None:
                        s.event.synchronize()                # the consumer's copies out of this slot have run
                    self.gather(ch, s)
                    full_q.put(s)
                full_q.put(None)
            except BaseException as exc:                      # surface loader errors in the consumer
                full_q.put(exc)

        th = threading.Thread(target=produce, daemon=True)
        th.start()
        try:
            while True:
                s = full_q.get()
                if s is None:
                    break
                if isinstance(s, BaseException):
                    raise s
                yield s.batch
                if self.pin:
                    s.event = torch.cuda.Event()
                    s.event.record()
                free_q.put(s)
        finally:
            stop.set()
            free_q.put(self.slots[0])
            th.join(timeout=5)
            if self.pin:
                # normal end or early break: the slot handed out last has no event yet -- make sure every copy out of
                # the staging ring has run before anybody (the next epoch's producer) rewrites it
                torch.cuda.current_stream().synchronize()
                for s in self.slots:
                    s.event = None
