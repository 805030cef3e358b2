"""Training-time forward / backward of a FullyConnected policy with two hidden layers as ONE
autograd node (the update of SURVEY.md section 8 row f1).

torch autograd runs the module as ~12 forward and ~25 backward kernels, most of them
elementwise passes over the [rows, H] activations (2 GB each at BASELINE config 2's
T x E x Np = 2.1 M rows): bias add, ReLU, three head GEMMs reading the same activations, two
softmaxes, their backward twins and the gradient accumulations between them.  Here the
GEMMs stay on cuBLAS (plain library GEMMs, float32 storage, TF32 only if the caller enabled
it globally) and everything between them is fused:
  * bias + ReLU ride in the GEMM epilogue (cuBLASLt through torch._addmm_activation),
  * the two action heads and the value head are ONE GEMM; `wdb_heads_softmax` turns its
    logits into dense per-head probabilities,
  * backward: `wdb_heads_softmax_backward` -> ONE GEMM for d(hidden), `wdb_relu_backward_bias`
    masks it in place and yields the bias gradient in the same pass.
Same math as fully_connected.py:51-89 under autograd (float32; sums in a different order).
"""
import torch
from torch.nn import functional as func

from warp_drive_b200 import lib as _lib


def _relu_backward_bias(dh, h):
    """dh *= (h > 0) in place; returns the column sums (the bias gradient)."""
    L = _lib.load()
    rows, width = dh.shape
    per = int(L.wdb_relu_backward_bias_rows(rows))
    partial = torch.empty((-(-rows // per), width), dtype=torch.float32, device=dh.device)
    _lib.check(L.wdb_relu_backward_bias(_lib.stream_ptr(), _lib.ptr(dh), _lib.ptr(h), rows,
                                        width, _lib.ptr(partial)), "relu_backward_bias")
    return partial.sum(0)


def _wgrad(a, b):
    """a^T b for a [rows, ka], b [rows, kb] (a weight gradient: the reduction runs over the
    batch rows).  cuBLAS picks a kernel for the single tall-skinny GEMM that reaches half of
    the HBM bandwidth; the same reduction as a batched GEMM over 16 row chunks plus a sum of
    the partials streams closer to the HBM peak (compare with scripts/gemm_variants.py)."""
    rows = a.shape[0]
    for chunks in (16, 8, 4, 2):
        if rows % chunks == 0 and rows // chunks >= 8192:
            ac = a.view(chunks, rows // chunks, a.shape[1])
            bc = b.view(chunks, rows // chunks, b.shape[1])
            return torch.bmm(ac.transpose(1, 2), bc).sum(0)
    return a.t().mm(b)


class _FusedMLPTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, obs, mask, w1, b1, w2, b2, wh0, bh0, wh1, bh1, wv, bv):
        L = _lib.load()
        rows, f = obs.shape
        a0 = wh0.shape[0]
        a1 = wh1.shape[0] if wh1 is not None else 0
        # Row pitches that are not a multiple of 16 bytes (71 observation features, 43 head
        # outputs) push cuBLAS onto its unaligned kernels (2-3x slower, measured): pad the
        # observation copy and the head GEMM to a multiple of 4 floats with zeros.
        fp = -(-f // 4) * 4
        if fp != f:
            padded = torch.empty((rows, fp), dtype=torch.float32, device=obs.device)
            _lib.check(L.wdb_pad_rows(_lib.stream_ptr(), _lib.ptr(obs), rows, f, fp,
                                      _lib.ptr(padded)), "pad_rows")
            obs = padded
            w1 = func.pad(w1, (0, fp - f))
        h1 = torch._addmm_activation(b1, obs, w1.t(), use_gelu=False)
        h2 = torch._addmm_activation(b2, h1, w2.t(), use_gelu=False)
        a = a0 + a1 + 1
        ap = _head_pitch(a0, a1)
        heads = [wh0] + ([wh1] if a1 else []) + [wv]
        biases = [bh0] + ([bh1] if a1 else []) + [bv]
        if ap != a:
            heads.append(torch.zeros((ap - a, wh0.shape[1]), dtype=wh0.dtype, device=wh0.device))
            biases.append(torch.zeros(ap - a, dtype=bh0.dtype, device=bh0.device))
        w3 = torch.cat(heads, 0)
        z3 = torch.addmm(torch.cat(biases, 0), h2, w3.t())
        p0 = torch.empty((rows, a0), dtype=torch.float32, device=obs.device)
        p1 = torch.empty((rows, a1), dtype=torch.float32, device=obs.device) if a1 else None
        values = torch.empty(rows, dtype=torch.float32, device=obs.device)
        if mask is None:
            _lib.check(L.wdb_heads_softmax(_lib.stream_ptr(), _lib.ptr(z3), rows, a0, a1, ap,
                                           _lib.ptr(p0), _lib.ptr(p1), _lib.ptr(values)),
                       "heads_softmax")
        else:
            # masked probabilities are exactly 0, so the unmasked backward gives them a zero
            # logit gradient
            _lib.check(L.wdb_heads_softmax_masked(
                _lib.stream_ptr(), _lib.ptr(z3), rows, a0, a1, ap, _lib.ptr(mask), a0 + a1,
                _lib.ptr(p0), _lib.ptr(p1), _lib.ptr(values)), "heads_softmax_masked")
        ctx.save_for_backward(obs, h1, h2, p0, p1 if a1 else p0, w2, w3)
        ctx.a0, ctx.a1, ctx.f = a0, a1, f
        if a1:
            return p0, p1, values
        return p0, values

    @staticmethod
    def backward(ctx, *grads):
        L = _lib.load()
        obs, h1, h2, p0, p1, w2, w3 = ctx.saved_tensors
        a0, a1, f = ctx.a0, ctx.a1, ctx.f
        g0, gv = grads[0], grads[-1]
        g1 = grads[1] if a1 else None
        rows = obs.shape[0]
        dz3 = torch.empty((rows, w3.shape[0]), dtype=torch.float32, device=obs.device)
        cont = lambda t: None if t is None else t.contiguous().float()   # noqa: E731
        g0, g1, gv = cont(g0), cont(g1), cont(gv)
        _lib.check(L.wdb_heads_softmax_backward(
            _lib.stream_ptr(), _lib.ptr(p0), _lib.ptr(p1 if a1 else None), _lib.ptr(g0),
            _lib.ptr(g1), _lib.ptr(gv), rows, a0, a1, w3.shape[0], _lib.ptr(dz3)),
            "heads_softmax_backward")
        dw3 = _wgrad(dz3, h2)
        db3 = dz3.sum(0)
        dh2 = dz3.mm(w3)
        db2 = _relu_backward_bias(dh2, h2)
        dw2 = _wgrad(dh2, h1)
        dh1 = dh2.mm(w2)
        del dh2
        db1 = _relu_backward_bias(dh1, h1)
        dw1 = _wgrad(dh1, obs)[:, :f]
        dwh0, dbh0 = dw3[:a0], db3[:a0]
        dwh1 = dw3[a0:a0 + a1] if a1 else None
        dbh1 = db3[a0:a0 + a1] if a1 else None
        dwv, dbv = dw3[a0 + a1:a0 + a1 + 1], db3[a0 + a1:a0 + a1 + 1]
        return None, None, dw1, db1, dw2, db2, dwh0, dbh0, dwh1, dbh1, dwv, dbv


def _head_pitch(a0, a1):
    """Row pitch of the head GEMM's logits: both heads and the value column, padded to 4."""
    return -(-(a0 + a1 + 1) // 4) * 4


def supported(model, obs, mask=None):
    """Two hidden layers, one or two softmax heads that both softmax kernels take (the
    library's own launch check), float32 CUDA tensors; an action mask, if any, has one row of
    every head's actions per observation row."""
    if getattr(model, "is_deterministic", True) or len(model.fc) != 2:
        return False
    if getattr(model, "is_recurrent", False):     # (a memoryless node)
        return False
    if len(model.output_dims) not in (1, 2):
        return False
    if not obs.is_cuda or obs.dtype != torch.float32 or obs.requires_grad:
        return False
    if mask is not None and (not mask.is_cuda or mask.requires_grad
                             or tuple(mask.shape) != tuple(obs.shape[:-1]) + (
                                 sum(int(a) for a in model.output_dims),)):
        return False
    a0 = int(model.output_dims[0])
    a1 = int(model.output_dims[1]) if len(model.output_dims) == 2 else 0
    if not _lib.load().wdb_heads_softmax_supported(a0, a1, _head_pitch(a0, a1)):
        return False
    return all(p.is_cuda and p.dtype == torch.float32 for p in model.parameters())


def fused_train_forward(model, obs, mask=None):
    """FullyConnected.forward(obs, action_mask=mask) -> ([probs per head], values) through the
    fused node."""
    lead = obs.shape[:-1]
    if getattr(model, "normalize_observations", False):
        obs = model.normalized_input(obs)
    x = obs.reshape(-1, obs.shape[-1])
    if not x.is_contiguous():
        x = x.contiguous()
    if mask is not None:
        mask = mask.reshape(x.shape[0], -1).float().contiguous()
    l1, l2 = model.fc["0"][0], model.fc["1"][0]
    h0 = model.policy_head[0]
    two = len(model.output_dims) == 2
    h1 = model.policy_head[1] if two else None
    out = _FusedMLPTrain.apply(
        x, mask, l1.weight, l1.bias, l2.weight, l2.bias, h0.weight, h0.bias,
        h1.weight if two else None, h1.bias if two else None,
        model.vf_head.weight, model.vf_head.bias)
    probs = [out[0].view(*lead, -1)] + ([out[1].view(*lead, -1)] if two else [])
    return probs, out[-1].view(*lead)
