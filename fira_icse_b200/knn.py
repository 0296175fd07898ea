"""Nearest-neighbour decoding (kNN-LM / kNN-MT, Khandelwal et al., ICLR 2020 / ICLR 2021): a trained model's
pointer mixture P mixed with the next words of the training positions whose decoder states are closest.

A `Datastore` holds one entry per target position of some commits (build_datastore): the decoder row at that position
as the key (bf16, 256 wide), its squared norm, and the word that came next as the value.  At every decoding position the
decoder row of each slot is the query; fira_knn_search returns its k nearest keys (exact, smallest (d_i, i) with
d_i = |q|^2 + norm_i - 2 q . key_i), and fira_pointer_mix_knn rewrites the model's triple so that the step kernels
decode from

    P'_j = (1 - lam) P_j + lam q_j  (j < V),   P'_{V+s} = (1 - lam) P_{V+s},
    q_w  = sum over neighbours i with word w of exp(-(d_i - d_1) / tau) / sum_i exp(-(d_i - d_1) / tau).

The neighbour mass goes to the vocabulary label of a word only; a copy label spelling the same word keeps the model's
probability alone (the diverse penalty and the rules already treat a copy and its vocabulary id as one word).  A
`KNNModel` is accepted wherever the decoding loop accepts a model -- sample.sample / score, beam.nbest (diverse groups
and lexical constraints too), mbr.mbr -- and every emitted token log-probability is log(clamp(P'_j, 1e-10, 1)).  This
needs no training: a datastore built from any DataSet directory (a team's own history) adapts a trained checkpoint to
it.  The reference-exact beam.beam_search, scst.scst_step, distill.distill_step and a KNNModel over an Ensemble are not
supported.
"""
import hashlib
import math
import numbers
import weakref

import torch

from . import ops
from ._lib import FIRA_BF16, FIRA_F32, call
from .ensemble import Ensemble
from .incremental import weights_key
from .model import TransModel

D = 256                   # key width (the decoder's model dimension)
MAX_K = 64                # fira_knn_search / fira_pointer_mix_knn
FORMAT = "fira-knn-datastore-1"

_FP = weakref.WeakKeyDictionary()      # model -> (weights_key, fingerprint)


def state_fingerprint(state_dict):
    """SHA-256 (hex) of a state_dict: names, shapes, dtypes and values, in order."""
    h = hashlib.sha256()
    for name, t in state_dict.items():
        t = t.detach().to("cpu").contiguous()
        h.update(f"{name}:{tuple(t.shape)}:{t.dtype};".encode())
        h.update(t.view(-1).view(torch.uint8).numpy().tobytes() if t.numel() else b"")
    return h.hexdigest()


def fingerprint(model):
    """state_fingerprint of the model's weights.  Keys built by another checkpoint lie in another space, so a datastore
    records the fingerprint of the model that built it.  Cached per weights_key."""
    wk = weights_key(model, model.decoder)
    cur = _FP.get(model)
    if cur is None or cur[0] != wk:
        cur = _FP[model] = (wk, state_fingerprint(model.state_dict()))
    return cur[1]


class Datastore:
    """keys [N, 256] bf16, norms [N] fp32, words [N] int32 (vocabulary ids), source [N, 2] int32 (dataset index of the
    commit, target position t; provenance only, the search does not read it), all on one device, plus the
    vocabulary size, the precision ('fp32' / 'bf16') and the fingerprint of the model that built it.  ValueError for a
    wrong dtype, shape or device, an empty store, N >= 2^31 or a word outside [0, vocab_size)."""

    def __init__(self, keys, norms, words, source, *, vocab_size, precision, fingerprint):
        for name, t, dt in (("keys", keys, torch.bfloat16), ("norms", norms, torch.float32),
                            ("words", words, torch.int32), ("source", source, torch.int32)):
            if not torch.is_tensor(t) or t.dtype != dt:
                raise ValueError(f"datastore {name} must be a {dt} tensor, got {getattr(t, 'dtype', type(t))}")
        if keys.dim() != 2 or keys.shape[1] != D:
            raise ValueError(f"datastore keys must have shape [N, {D}], got {tuple(keys.shape)}")
        N = keys.shape[0]
        if not 1 <= N < 2 ** 31:
            raise ValueError(f"a datastore needs 1 <= N < 2^31 entries, got {N}")
        if tuple(norms.shape) != (N,) or tuple(words.shape) != (N,) or tuple(source.shape) != (N, 2):
            raise ValueError(f"datastore norms / words must be [N = {N}] and source [N, 2], got {tuple(norms.shape)}, "
                             f"{tuple(words.shape)}, {tuple(source.shape)}")
        if len({t.device for t in (keys, norms, words, source)}) != 1:
            raise ValueError("datastore tensors must be on one device")
        if isinstance(vocab_size, bool) or not isinstance(vocab_size, int) or vocab_size < 1:
            raise ValueError(f"vocab_size must be a positive integer, got {vocab_size!r}")
        if precision not in ("fp32", "bf16"):
            raise ValueError(f"precision must be 'fp32' or 'bf16', got {precision!r}")
        if not isinstance(fingerprint, str) or not fingerprint:
            raise ValueError("a datastore needs the fingerprint of the model that built it")
        if bool(((words < 0) | (words >= vocab_size)).any()):
            raise ValueError(f"datastore words must be vocabulary ids in [0, {vocab_size})")
        self.keys, self.norms = keys.contiguous(), norms.contiguous()
        self.words, self.source = words.contiguous(), source.contiguous()
        self.vocab_size, self.precision, self.fingerprint = vocab_size, precision, fingerprint

    @property
    def N(self):
        return self.keys.shape[0]

    @property
    def device(self):
        return self.keys.device

    @property
    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.keys, self.norms, self.words, self.source))

    def to(self, device):
        """The same datastore on `device`."""
        return Datastore(*(t.to(device) for t in (self.keys, self.norms, self.words, self.source)),
                         vocab_size=self.vocab_size, precision=self.precision, fingerprint=self.fingerprint)

    def save(self, path):
        torch.save({"format": FORMAT, "d": D, "vocab_size": self.vocab_size, "precision": self.precision,
                    "fingerprint": self.fingerprint, "keys": self.keys.cpu(), "norms": self.norms.cpu(),
                    "words": self.words.cpu(), "source": self.source.cpu()}, path)

    @classmethod
    def load(cls, path, device, *, vocab_size=None, precision=None):
        """The datastore saved at `path`, on `device`.  ValueError for another file format, another key width, and a
        vocabulary size or precision other than the given ones (None: not checked)."""
        s = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(s, dict) or s.get("format") != FORMAT:
            raise ValueError(f"{path} is not a kNN datastore ({FORMAT})")
        if s["d"] != D:
            raise ValueError(f"{path}: key width {s['d']}, expected {D}")
        if vocab_size is not None and s["vocab_size"] != vocab_size:
            raise ValueError(f"{path}: vocab_size {s['vocab_size']}, the model has {vocab_size}")
        if precision is not None and s["precision"] != precision:
            raise ValueError(f"{path}: built in {s['precision']}, the model runs in {precision}")
        return cls(*(s[k].to(device) for k in ("keys", "norms", "words", "source")), vocab_size=s["vocab_size"],
                   precision=s["precision"], fingerprint=s["fingerprint"])


@torch.no_grad()
def build_datastore(model, batches, *, first_index, start_id, eos_id, pad_id, unk_id):
    """A Datastore from padded batches (the 8-tuples of run_model.py: sou, tar, attr, mark, ast_change, edge, tar_label,
    sub_token), in eval mode and the model's own precision.  first_index: dataset index of the first batch's first
    commit; the batches follow one another.  For commit b and position t with shifted label y != 0 (y =
    TransModel.shifted_label(tar_label)[b, t]): word = y if y < V, else copy_src[b, y - V] (copy_src = cat(sou,
    sub_token)); entries whose word is pad_id, <start> or <unkm> are dropped, <eos> entries are kept (neighbours can end
    a message).  key = the teacher-forced decoder row (b, t) in bf16, norm = sum key^2 in fp32."""
    from .decode_loop import encode
    from . import optim as _optim
    if not isinstance(model, TransModel):
        raise TypeError(f"build_datastore takes a TransModel, got {type(model).__name__}")
    model.eval()
    if model.precision == "bf16":
        _optim.ensure_fresh(model)
    V = model.vocab_size
    dev = model.out_fc.weight.device
    parts, first = [], int(first_index)
    for batch in batches:
        sou, tar, _, mark, ast_change, edge, tar_label, sub_token = batch
        B = sou.shape[0]
        memory, mem_mask, copy_src = encode(model, sou, mark, ast_change, edge, sub_token, pad_id)
        tar = tar.to(dev)
        dec = model.decoder(tar, memory, mem_mask, tar != 0)                    # [B, T, D]
        label = TransModel.shifted_label(tar_label.to(dev)).long()
        T, S = label.shape[1], copy_src.shape[1]
        word = torch.where(label < V, label, copy_src.long().gather(1, (label - V).clamp(0, S - 1)))
        keep = (label != 0) & (word != pad_id) & (word != start_id) & (word != unk_id)
        b, t = keep.nonzero(as_tuple=True)
        keys = dec[b, t].to(torch.bfloat16)
        parts.append((keys, keys.float().square().sum(1), word[b, t].to(torch.int32),
                      torch.stack((b + first, t), 1).to(torch.int32)))
        first += B
    if not parts:
        raise ValueError("build_datastore: no batches")
    keys, norms, words, source = (torch.cat(x) for x in zip(*parts))
    if bool(((words < 0) | (words >= V)).any()):
        raise ValueError("build_datastore: a copied word is not a vocabulary id")
    return Datastore(keys, norms, words, source, vocab_size=V, precision=model.precision,
                     fingerprint=fingerprint(model))


def check_settings(k, temperature, lam, N=None):
    """ValueError for k outside [1, min(64, N)], a temperature that is not positive and finite, or lam outside (0, 1)
    (lam = 0 is the plain model, lam = 1 leaves every word without a neighbour at exactly 0)."""
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= MAX_K:
        raise ValueError(f"k must be an integer in [1, {MAX_K}], got {k!r}")
    if N is not None and k > N:
        raise ValueError(f"k = {k} exceeds the datastore's {N} entries")
    if isinstance(temperature, bool) or not isinstance(temperature, numbers.Real) or \
            not 0.0 < float(temperature) < math.inf:
        raise ValueError(f"temperature must be positive and finite, got {temperature!r}")
    if isinstance(lam, bool) or not isinstance(lam, numbers.Real) or not 0.0 < float(lam) < 1.0:
        raise ValueError(f"lam must be in (0, 1), got {lam!r}")


class KNNModel:
    """model: a TransModel; datastore: a Datastore it built (the same fingerprint); k neighbours, temperature tau and
    interpolation weight lam (module docstring).  The defaults are common starting points of the kNN-MT papers, not
    tuned on this data.  Checked on the host before any device work: TypeError for another model type (an Ensemble is
    not supported), ValueError for the settings, k > N, another device, vocabulary, precision or fingerprint.  The
    decoding loops cached for it hold the datastore and a search workspace while the model lives;
    decode_loop.drop_loops(knn_model) releases them."""

    def __init__(self, model, datastore, k=8, temperature=10.0, lam=0.25):
        if isinstance(model, Ensemble):
            raise TypeError("a KNNModel over an Ensemble is not supported: wrap a single TransModel")
        if not isinstance(model, TransModel):
            raise TypeError(f"model must be a TransModel, got {type(model).__name__}")
        if not isinstance(datastore, Datastore):
            raise TypeError(f"datastore must be a Datastore, got {type(datastore).__name__}")
        check_settings(k, temperature, lam, datastore.N)
        dev = model.out_fc.weight.device
        if dev.type != "cuda" or datastore.device != dev:
            raise ValueError(f"the model is on {dev}, the datastore on {datastore.device}: both must be on one CUDA device")
        if datastore.vocab_size != model.vocab_size:
            raise ValueError(f"the datastore has vocab_size {datastore.vocab_size}, the model {model.vocab_size}")
        if datastore.precision != model.precision:
            raise ValueError(f"the datastore was built in {datastore.precision}, the model runs in {model.precision}")
        if fingerprint(model) != datastore.fingerprint:
            raise ValueError("the datastore was built by other weights than this model's (fingerprint mismatch)")
        self.model, self.datastore = model, datastore
        self.k, self.temperature, self.lam = k, float(temperature), float(lam)

    def eval(self):
        self.model.eval()
        return self

    @property
    def precision(self):
        return self.model.precision

    @property
    def vocab_size(self):
        return self.model.vocab_size

    @property
    def device(self):
        return self.model.out_fc.weight.device


def base_model(model):
    """The TransModel (or Ensemble) a KNNModel wraps, or the model itself."""
    return model.model if isinstance(model, KNNModel) else model


def workspace_bytes(R, k, device):
    """fira_knn_search's workspace for the full key split: 8 k max(R, 128 SMs) bytes (include/fira_b200.h)."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    return 8 * k * max(R, 128 * sms)


def search_into(datastore, queries, k, workspace, idx, dist):
    """fira_knn_search of queries [R, >= 256] (fp32 or bf16, row stride a multiple of 8) into idx [R, k] int32 and
    dist [R, k] fp32 on the current stream (capturable)."""
    R = queries.shape[0]
    code = FIRA_BF16 if queries.dtype == torch.bfloat16 else FIRA_F32
    p = ops._ptr
    call("fira_knn_search", p(queries), queries.stride(0), code, p(datastore.keys), p(datastore.norms), datastore.N, R,
         k, p(workspace), workspace.numel(), p(idx), p(dist), ops._stream())


@torch.no_grad()
def search(datastore, queries, k):
    """The k nearest entries of each query row -> (idx [R, k] int64, dist [R, k] fp32), ascending (d_i, i).
    queries: [R, 256] fp32 or bf16 on the datastore's device (rounded to bf16).  ValueError for a bad k or query."""
    check_settings(k, 1.0, 0.5, datastore.N)
    if not torch.is_tensor(queries) or queries.dtype not in (torch.float32, torch.bfloat16) or queries.dim() != 2 \
            or queries.shape[1] != D:
        raise ValueError(f"queries must be a [R, {D}] fp32 or bf16 tensor")
    if queries.device != datastore.device:
        raise ValueError(f"queries are on {queries.device}, the datastore on {datastore.device}")
    q = queries.contiguous()
    R = q.shape[0]
    idx = torch.empty((R, k), dtype=torch.int32, device=q.device)
    dist = torch.empty((R, k), dtype=torch.float32, device=q.device)
    if R:
        ws = torch.empty(workspace_bytes(R, k, q.device), dtype=torch.uint8, device=q.device)
        search_into(datastore, q, k, ws, idx, dist)
    return idx.long(), dist
