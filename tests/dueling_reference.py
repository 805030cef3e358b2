"""Float64 NumPy reference of the dueling head's fold and of the unfold of its gradients
(include/wdb200.h wdb_dueling_*; models/fully_connected_q.py DuelingHead)."""
import numpy as np


def stream_params(head):
    """{name: float64 array} of a DuelingHead's stream parameters: value_/adv_ + hw, hb (S > 0),
    ow, ob."""
    (vh, vo), (ah, ao) = head.streams()
    out = {}
    for prefix, hidden, output in (("value_", vh, vo), ("adv_", ah, ao)):
        layers = ([("h", hidden)] if hidden is not None else []) + [("o", output)]
        for name, layer in layers:
            out[prefix + name + "w"] = layer.weight.detach().cpu().double().numpy()
            out[prefix + name + "b"] = layer.bias.detach().cpu().double().numpy()
    return out


def _centred(x, A, N):
    y = x.reshape(A, N, *x.shape[1:])
    return (y - y.mean(axis=0, keepdims=True)).reshape(x.shape)


def fold(p, A, N, S):
    """[(weight, bias)] of the folded layers: [hidden (S > 0),] output."""
    vo, vob = p["value_ow"], p["value_ob"]
    ao, aob = p["adv_ow"], p["adv_ob"]
    b = np.tile(vob, A) + _centred(aob, A, N)
    if S == 0:
        return [(np.tile(vo, (A, 1)) + _centred(ao, A, N), b)]
    hidden = (np.concatenate([p["value_hw"], p["adv_hw"]]),
              np.concatenate([p["value_hb"], p["adv_hb"]]))
    return [hidden, (np.concatenate([np.tile(vo, (A, 1)), _centred(ao, A, N)], axis=1), b)]


def unfold(grads, A, N, S):
    """The stream parameters' gradients (names of stream_params) from the folded layers'
    gradients [(gw, gb)]: the transpose of the fold."""
    out = {}
    if S > 0:
        (ghw, ghb), (gow, gob) = grads
        out["value_hw"], out["adv_hw"] = ghw[:S], ghw[S:]
        out["value_hb"], out["adv_hb"] = ghb[:S], ghb[S:]
        gv, ga = gow[:, :S], gow[:, S:]
    else:
        (gow, gob), = grads
        gv = ga = gow
    out["value_ow"] = gv.reshape(A, N, -1).sum(0)
    out["value_ob"] = gob.reshape(A, N).sum(0)
    out["adv_ow"] = _centred(ga, A, N)
    out["adv_ob"] = _centred(gob, A, N)
    return out


def mlp(x, layers):
    """ReLU hidden layers, raw last layer (float64)."""
    for i, (w, b) in enumerate(layers):
        x = x @ w.T + b
        if i < len(layers) - 1:
            x = np.maximum(x, 0.0)
    return x
