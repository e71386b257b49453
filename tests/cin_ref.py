"""The float64 reference of the pooled CIN features that the native CIN entry points return: oracle.layers_ref.cin with
an identity output head.  The head only adds exact float64 zeros, so the result carries the bits of the oracle's
sum-pooled feature maps."""
import torch

from oracle import layers_ref as L


def cin_pooled_f64(x, sizes, direct, filters, biases, act):
    """x (B, F, D); filters[k] (F * H_k, L_k); biases a list of (L_k,) or None; act 1 = relu, 0 = linear.
    Returns (B, pooled width); differentiable in every tensor argument."""
    params = dict(cross_layer_size=sizes, direct=direct, use_bias=biases is not None,
                  activation='relu' if act else 'linear')
    width = L.cin_pooled_width(x.shape[1], params)
    w = {f'f_{k}': filters[k].unsqueeze(0) for k in range(len(sizes))}
    for k in range(len(sizes) if biases is not None else 0):
        w[f'bias{k}'] = biases[k]
    w['exFM_out/kernel'] = torch.eye(width, dtype=x.dtype)
    w['exFM_out/bias'] = torch.zeros(width, dtype=x.dtype)
    return L.cin(x, params, w)
