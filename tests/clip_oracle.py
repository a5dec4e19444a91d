"""fp32 functional restatement of transformers' CLIPTextModel (models/clip/modeling_clip.py, eager attention) for SD-1.5's
text encoder: the reference the native encoder is compared with.  No transformers import; each function names the code it
restates.  Works on any device and dtype (the tests run it in fp32 on the CPU or, with TF32 off, on the GPU)."""
from __future__ import annotations

import math

import torch

P = "text_model"


def quick_gelu(x):
    """activations.QuickGELUActivation: x * sigmoid(1.702 x)."""
    return x * torch.sigmoid(1.702 * x)


def embeddings(sd, ids):
    """CLIPTextEmbeddings.forward: token_embedding(ids) + position_embedding(arange(L))."""
    L = ids.shape[1]
    return sd[f"{P}.embeddings.token_embedding.weight"][ids] + sd[f"{P}.embeddings.position_embedding.weight"][:L]


def linear(x, sd, name):
    return x @ sd[name + ".weight"].t() + sd[name + ".bias"]


def layer_norm(x, sd, name, eps=1e-5):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], eps)


def attention(x, sd, name, heads):
    """CLIPAttention.forward with eager_attention_forward: softmax(q k^T * d^-0.5 + causal mask) v, then out_proj.  The
    causal mask (_create_4d_causal_attention_mask) puts the dtype's minimum above the diagonal; -inf is the same after
    the softmax."""
    n, L, C = x.shape
    d = C // heads
    q, k, v = (linear(x, sd, f"{name}.{t}_proj").view(n, L, heads, d).transpose(1, 2) for t in "qkv")
    s = (q @ k.transpose(-1, -2)) * d ** -0.5
    mask = torch.triu(torch.ones(L, L, dtype=torch.bool, device=x.device), 1)
    p = torch.softmax(s.masked_fill(mask, -math.inf), dim=-1)
    o = (p @ v).transpose(1, 2).reshape(n, L, C)
    return linear(o, sd, f"{name}.out_proj")


def encoder_layer(x, sd, name, heads, eps=1e-5):
    """CLIPEncoderLayer.forward: pre-LN attention and MLP (fc2(quick_gelu(fc1))), each with a residual."""
    x = x + attention(layer_norm(x, sd, f"{name}.layer_norm1", eps), sd, f"{name}.self_attn", heads)
    h = layer_norm(x, sd, f"{name}.layer_norm2", eps)
    return x + linear(quick_gelu(linear(h, sd, f"{name}.mlp.fc1")), sd, f"{name}.mlp.fc2")


def text_model(sd, ids, layers=12, heads=12, eps=1e-5):
    """CLIPTextTransformer.forward -> (last_hidden_state after final_layer_norm, the layers + 1 hidden states before it)."""
    x = embeddings(sd, ids)
    hidden = [x]
    for i in range(layers):
        x = encoder_layer(x, sd, f"{P}.encoder.layers.{i}", heads, eps)
        hidden.append(x)
    return layer_norm(x, sd, f"{P}.final_layer_norm", eps), hidden
