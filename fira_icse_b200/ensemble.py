"""Ensemble decoding: several checkpoints decoded as one model whose distribution is the weighted average of theirs.

    P_j = sum_m w_m P^m_j        (P^m the dual-copy mixture of member m, Model.py:54-86; sum_m w_m = 1)

This is fairseq's rule (an average of probabilities, not of log-probabilities).  Every decoder of decode_loop's
position loop -- sample.sample / score, beam.nbest (diverse groups included), mbr.mbr -- accepts an `Ensemble` where
it accepts a model and applies its own rule to P: temperature, top-k and top-p act on log P, the beam rankings and
their length penalty use P, prefixes, n-gram blocking and the minimum length apply as for one model, and every emitted
token log-probability is log(clamp(P_j, 1e-10, 1)), so sample.score of an ensemble is log P(message | commit).

Each position runs every member's decoder row and output head, then fira_pointer_mix_ensemble rewrites the M
(logits, copy scores, gate logits) triples into one fp32 triple whose mixture is P (include/fira_b200.h), and the
unchanged step kernel reads that triple, all inside the position's CUDA graph.  The reference-exact beam.beam_search
and scst.scst_step take a single model only.
"""
import math
import numbers

from .model import TransModel

MAX_MEMBERS = 8           # fira_pointer_mix_ensemble passes the members' pointers in its launch parameters


class Ensemble:
    """models: 1..8 TransModel on one CUDA device, one precision and one vocabulary (the same object may appear more
    than once); weights: None (uniform) or M positive finite numbers, normalised in float64 to sum to 1.  Checked on
    the host: ValueError / TypeError before any device work."""

    def __init__(self, models, weights=None):
        if isinstance(models, TransModel) or not isinstance(models, (list, tuple)):
            raise TypeError(f"models must be a list or tuple of TransModel, got {type(models).__name__}")
        models = tuple(models)
        if not 1 <= len(models) <= MAX_MEMBERS:
            raise ValueError(f"an ensemble takes 1 to {MAX_MEMBERS} models, got {len(models)}")
        for i, m in enumerate(models):
            if not isinstance(m, TransModel):
                raise TypeError(f"member {i} is a {type(m).__name__}, not a TransModel")
        M = len(models)
        if weights is None:
            weights = [1.0] * M
        if isinstance(weights, (str, bytes)) or not hasattr(weights, "__len__"):
            raise TypeError(f"weights must be None or a sequence of {M} numbers, got {type(weights).__name__}")
        weights = list(weights)
        if len(weights) != M:
            raise ValueError(f"{M} models need {M} weights, got {len(weights)}")
        for w in weights:
            if isinstance(w, bool) or not isinstance(w, numbers.Real):
                raise TypeError(f"weights must be numbers, got {w!r}")
            if not 0.0 < float(w) < math.inf:
                raise ValueError(f"weights must be positive and finite, got {w!r}")
        first = models[0]
        for i, m in enumerate(models[1:], 1):
            if m.precision != first.precision:
                raise ValueError(f"member {i} has precision {m.precision!r}, member 0 {first.precision!r}")
            if m.vocab_size != first.vocab_size:
                raise ValueError(f"member {i} has vocab_size {m.vocab_size}, member 0 {first.vocab_size}")
            if m.out_fc.weight.device != first.out_fc.weight.device:
                raise ValueError(f"member {i} is on {m.out_fc.weight.device}, member 0 on {first.out_fc.weight.device}")
        if first.out_fc.weight.device.type != "cuda":
            raise ValueError(f"ensemble members must be on a CUDA device, got {first.out_fc.weight.device}")
        total = math.fsum(float(w) for w in weights)
        self.models = models
        self.weights = tuple(float(w) / total for w in weights)
        self.log_weights = tuple(math.log(w) for w in self.weights)

    def __len__(self):
        return len(self.models)

    def eval(self):
        """Every member in evaluation mode (decoding runs without dropout) -> self."""
        for m in self.models:
            m.eval()
        return self

    @property
    def precision(self):
        return self.models[0].precision

    @property
    def vocab_size(self):
        return self.models[0].vocab_size

    @property
    def device(self):
        return self.models[0].out_fc.weight.device


def members(model):
    """The models an Ensemble averages, or (model,) for one model."""
    return model.models if isinstance(model, Ensemble) else (model,)


def refuse(model, what):
    """TypeError for an Ensemble or a knn.KNNModel passed where only one model is supported."""
    from .knn import KNNModel
    if isinstance(model, Ensemble):
        raise TypeError(f"{what} takes a single model; ensembles decode through sample, score, nbest and mbr")
    if isinstance(model, KNNModel):
        raise TypeError(f"{what} takes a single model; a KNNModel decodes through sample, score, nbest and mbr")
