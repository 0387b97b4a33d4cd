"""Restatement of the engine's dropout mask (include/pertgnn.h, pert_model_forward) and an oracle forward that takes
prescribed dropout masks.  Shared by tests/test_dropout_rng.py (CPU) and tests/test_gpu_dropout.py."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.model_oracle import global_add_pool

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Random123).  ctr: four uint32 values or arrays (broadcast), key: two ints -> four uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M32 for c in ctr)
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
        p0 = np.uint64(0xD2511F53) * c0          # < 2^64: exact in uint64
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def threshold(p):
    """T = floor(p * 2^32) in fp64 of the float32 rate the C-ABI receives (2^32 at p = 1: nothing kept)."""
    return math.floor(float(np.float32(p)) * 4294967296.0)


def scale_of(p):
    p32 = float(np.float32(p))
    return 0.0 if p32 >= 1.0 else float(np.float32(1.0 / (1.0 - p32)))


def dropout_mask(seed, step, layer, N, H, p):
    """bool [N, H]: the keep mask of BatchNorm layer ``layer`` at the counter (seed, step)."""
    seed = int(seed) & (2 ** 64 - 1)
    step = int(step) & (2 ** 64 - 1)
    g = np.arange(N * H // 4, dtype=np.uint64)
    w = philox4x32_10((g, layer, step & 0xFFFFFFFF, step >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    words = np.stack(w, axis=1).reshape(N, H)     # group g = row*(H/4) + col/4, word j -> column col + j
    return words.astype(np.uint64) >= np.uint64(threshold(p))


def dropout_masks(seed, step, N, H, p, n_bn):
    return {f"bn{l}": torch.from_numpy(dropout_mask(seed, step, l, N, H, p)) for l in range(n_bn)}


def oracle_forward(oracle, x, cat_X, edge_index, edge_attr, pattern_num_nodes, pattern_probs, entry_id, batch,
                   relu_masks=None, dropout_masks=None, capture=None):
    """``OracleSAGEDeterministic.forward`` (reference model.py:76-114) with the dropout after every BatchNorm + ReLU
    either torch's ``F.dropout`` (``dropout_masks`` None, as the oracle does) or ``t * mask / (1 - p)`` with the given
    {'bn{i}': bool [N,H]} masks (zero at p = 1).  ``relu_masks`` as in the oracle.  ``capture`` (dict or None)
    receives the BatchNorm + ReLU outputs before dropout as 'bn{i}'."""
    p = oracle.dropout
    relu = (lambda t, k: F.relu(t)) if relu_masks is None else (lambda t, k: t * relu_masks[k].to(t.dtype))
    cat_embeds = 0
    for i, emb in enumerate(oracle.cat_embedding):
        cat_embeds = cat_embeds + emb(cat_X[:, i])
    x = torch.cat([x, cat_embeds], dim=1)
    edge_embeds = torch.cat([oracle.interface_embeds(edge_attr[:, 0]), oracle.rpctype_embeds(edge_attr[:, 1])], dim=1)
    for i, conv in enumerate(oracle.convs[:-1]):
        x = relu(oracle.bns[i](conv(x, edge_index, edge_embeds)), f"bn{i}")
        if capture is not None:
            capture[f"bn{i}"] = x.detach()
        if dropout_masks is None:
            x = F.dropout(x, p=p, training=oracle.training)
        elif oracle.training:
            x = x * 0.0 if p >= 1.0 else x * dropout_masks[f"bn{i}"].to(x.dtype) / (1.0 - p)
    x = oracle.convs[-1](x, edge_index, edge_embeds)
    local_predict = oracle.local_linear(x)
    x = x * pattern_probs / pattern_num_nodes
    g = torch.cat([global_add_pool(x, batch), oracle.entry_embeds(entry_id)], dim=1)
    g = oracle.global_linear2(relu(oracle.global_linear1(g), "head"))
    return g, local_predict
