"""High-precision references and error bars for the step engine's own kernels (csrc/engine.cu): the fused global head
(``k_head_fwd`` / ``k_head_bwd``), the grouped small GEMMs of the edge tables (``k_small_gemm``) and the parameter pack /
gradient unpack (``k_pack`` / ``k_unpack``).

Every reference takes the kernel's own float32 inputs -- the engine's intermediates read from the workspace
(``pert_model_workspace_offset``) and the flat parameter buffer -- and computes in float64.  All of them work in the
engine's layout: width Hp = pert_model_width(H), the padded copies zero in rows / columns [H, Hp), global_linear1 as
[Hp, 2Hp] with its [pool | entry] column blocks at 0 and Hp.

u = 2^-24 is the unit roundoff of float32 and gamma(n) = n u / (1 - n u).  A sum whose every term passes through at
most n float32 roundings (an FMA, an addition or an atomic addition each round once) is within gamma(n) * sum |terms| of
the exact sum, whatever the order of the additions (Higham, Accuracy and Stability of Numerical Algorithms, 3.1).  So
every bar is a worst-case bound, ``gamma(n) * (|A| |B|)``, with n the longest chain of the kernel's summation order;
the derivation sits next to each bar, and no order of the atomic additions can push an error past it.

``*_f32`` are numpy float32 restatements of the kernels' summation orders, with switches for the defects the bars must
catch (tests/test_engine_parts_ref.py)."""
import math

import numpy as np
import torch

U = 2.0 ** -24
F32 = np.float32
HEAD_G = 8                        # graphs per CTA of k_head_fwd / k_head_bwd
HEAD_SMEM_MAX = 200 * 1024        # engine.cu: head_slice's shared-memory budget
PROJ = ("lin_query", "lin_key", "lin_value", "lin_skip")   # the four row blocks q | k | v | skip of W4


def gamma(n):
    return n * U / (1.0 - n * U)


def al64(n):
    return (max(int(n), 1) + 63) // 64 * 64


def worst(got, ref, bar):
    """Largest |got - ref| / bar (<= 1 passes).  Where the bar is 0 the kernel must be exact: any difference there
    counts as infinitely far."""
    got, ref, bar = (torch.as_tensor(t).double() for t in (got, ref, bar))
    err = (got - ref).abs()
    if err.numel() == 0:
        return 0.0
    r = torch.where(bar > 0, err / torch.where(bar > 0, bar, torch.ones_like(bar)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    return float(r.max())


def head_slice(full, per_unit, fixed):
    """engine.cu head_slice: the widest slice of W1 (halved while it does not fit) within the shared-memory budget."""
    s = full
    while s % 8 == 0 and (per_unit * s + fixed) * 4 > HEAD_SMEM_MAX:
        s //= 2
    return s


def fwd_slice(Hp):
    """Rows of W1 one forward stage holds (k_head_fwd's ns)."""
    return head_slice(Hp, 2 * Hp, HEAD_G * 2 * Hp)


def bwd_slice(Hp):
    """Columns of W1 one backward stage holds (k_head_bwd's cs)."""
    return head_slice(2 * Hp, Hp, HEAD_G * 3 * Hp)


# ------------------------------------------------------------------------------------------------------ layouts
def _mat(flat, off, rows, cols):
    return flat[off:off + rows * cols].view(rows, cols)


def _pad(t, shape):
    out = torch.zeros(shape, dtype=t.dtype)
    out[tuple(slice(0, s) for s in t.shape)] = t
    return out


def pad_w1(W1, Hp, entry_col=None):
    """global_linear1.weight [H, 2H] -> the engine's [Hp, 2Hp]: pool columns at 0, entry columns at ``entry_col``
    (Hp; a defective copy may put them elsewhere)."""
    H = W1.shape[0]
    c = Hp if entry_col is None else entry_col
    out = torch.zeros(Hp, 2 * Hp, dtype=W1.dtype)
    out[:H, :H] = W1[:, :H]
    out[:H, c:c + H] = W1[:, H:]
    return out


def head_params(d, Hp, flat):
    """(W1 [Hp, 2Hp], b1 [Hp], W2 [Hp], b2 [1], entry table [n_entry, Hp]) as k_head_* read them."""
    H = d.H
    return (pad_w1(_mat(flat, d.off_g1_w, H, 2 * H), Hp), _pad(flat[d.off_g1_b:d.off_g1_b + H], (Hp,)),
            _pad(flat[d.off_g2_w:d.off_g2_w + H], (Hp,)), flat[d.off_g2_b:d.off_g2_b + 1].clone(),
            _pad(_mat(flat, d.off_entry, d.n_entry, H), (d.n_entry, Hp)))


def edge_params(d, Hp, flat, l):
    """(if_emb [n_if, Hp], rpc_emb [n_rpc, Hp], WeA [Hp, Hp], WeB [Hp, Hp]) of conv l, zero-padded."""
    H = d.H
    We = _mat(flat, d.off_we[l], H, 2 * H)
    return (_pad(_mat(flat, d.off_if, d.n_if, H), (d.n_if, Hp)), _pad(_mat(flat, d.off_rpc, d.n_rpc, H), (d.n_rpc, Hp)),
            _pad(We[:, :H], (Hp, Hp)), _pad(We[:, H:], (Hp, Hp)))


def conv_pack(d, Hp, l, flat):
    """(W4 [4, Hp, K], b4 [4, Hp], WeA [Hp, Hp], WeB [Hp, Hp]) of conv l as append_layer_segs places them: conv 0's
    reference input order [x (F) | emb (H)] becomes [emb at 0 | x at Hp | pad], K = k0 for conv 0 and Hp after it."""
    H, F = d.H, d.F
    K = d.k0 if l == 0 else Hp
    Din = F + H if l == 0 else H
    w4 = torch.zeros(4, Hp, K)
    b4 = torch.zeros(4, Hp)
    offs_w = (d.off_wq[l], d.off_wk[l], d.off_wv[l], d.off_ws[l])
    offs_b = (d.off_bq[l], d.off_bk[l], d.off_bv[l], d.off_bs[l])
    for p in range(4):
        W = _mat(flat, offs_w[p], H, Din)
        if l == 0:
            w4[p, :H, :H] = W[:, F:]
            w4[p, :H, Hp:Hp + F] = W[:, :F]
        else:
            w4[p, :H, :H] = W
        b4[p, :H] = flat[offs_b[p]:offs_b[p] + H]
    _, _, weA, weB = edge_params(d, Hp, flat, l)
    return w4, b4, weA, weB


def padded_tensors(d, Hp, L, flat):
    """The zero-padded copies (Hp > H) in carve()'s order: categorical tables, entry, interface and rpc tables,
    BatchNorm gamma / beta of each BatchNorm, local_linear, global_linear1, its bias, global_linear2."""
    H = d.H
    out = [_pad(_mat(flat, d.off_cat[i], d.cat_rows[i], H), (d.cat_rows[i], Hp)) for i in range(d.n_cat)]
    out += [_pad(_mat(flat, o, n, H), (n, Hp)) for o, n in ((d.off_entry, d.n_entry), (d.off_if, d.n_if),
                                                            (d.off_rpc, d.n_rpc))]
    for l in range(L - 1):
        out += [_pad(flat[d.off_bn_g[l]:d.off_bn_g[l] + H], (Hp,)), _pad(flat[d.off_bn_b[l]:d.off_bn_b[l] + H], (Hp,))]
    out.append(_pad(flat[d.off_local_w:d.off_local_w + H], (Hp,)))
    W1, b1, W2, _, _ = head_params(d, Hp, flat)
    return out + [W1, b1, W2]


def packed_restatement(d, Hp, L, flat):
    """float32 [pert_model_packed_bytes / 4]: the packed region k_pack writes from ``flat``, slot by slot in carve()'s
    order, each slot padded to 64 floats: per conv W4, b4, W4^T [K, 4Hp], WeA, WeB and their transposes; then at
    Hp > H the padded copies."""
    parts = []

    def put(t):
        t = t.reshape(-1).float()
        parts.extend([t, torch.zeros(al64(t.numel()) - t.numel())])

    for l in range(L):
        w4, b4, weA, weB = conv_pack(d, Hp, l, flat)
        put(w4)
        put(b4)
        put(w4.reshape(4 * Hp, -1).T.contiguous())
        for t in (weA, weB, weA.T, weB.T):
            put(t.contiguous())
    if Hp != d.H:
        for t in padded_tensors(d, Hp, L, flat):
            put(t)
    return torch.cat(parts)


def packed_pad_mask(d, Hp, L, n_flat):
    """bool [pert_model_packed_bytes / 4]: True where the packed region holds padding (rows / columns [H, Hp), the
    conv-0 pad columns, the 64-float alignment tails): the slots packed_restatement leaves 0 from an all-ones buffer."""
    return packed_restatement(d, Hp, L, torch.ones(n_flat)) == 0


def conv_unpack(d, Hp, l, dw4, db4, dweA, dweB):
    """The packed gradients of conv l (workspace codes 8..11) in the reference's layout, as k_unpack adds them:
    {'lin_query.weight': [H, Din], ..., 'lin_skip.bias': [H], 'lin_edge.weight': [H, 2H]}."""
    H, F = d.H, d.F
    dw4 = dw4.reshape(4, Hp, -1)
    db4 = db4.reshape(4, Hp)
    out = {}
    for p, name in enumerate(PROJ):
        w = dw4[p, :H]
        out[f"{name}.weight"] = torch.cat([w[:, Hp:Hp + F], w[:, :H]], 1) if l == 0 else w[:, :H]
        out[f"{name}.bias"] = db4[p, :H]
    out["lin_edge.weight"] = torch.cat([dweA.reshape(Hp, Hp)[:H, :H], dweB.reshape(Hp, Hp)[:H, :H]], 1)
    return out


def conv_param_views(d, l, flat):
    """The same dict of conv l's parameters (or gradients) as views of a flat buffer."""
    H, F = d.H, d.F
    Din = F + H if l == 0 else H
    ow = (d.off_wq[l], d.off_wk[l], d.off_wv[l], d.off_ws[l])
    ob = (d.off_bq[l], d.off_bk[l], d.off_bv[l], d.off_bs[l])
    out = {}
    for p, name in enumerate(PROJ):
        out[f"{name}.weight"] = _mat(flat, ow[p], H, Din)
        out[f"{name}.bias"] = flat[ob[p]:ob[p] + H]
    out["lin_edge.weight"] = _mat(flat, d.off_we[l], H, 2 * H)
    return out


# ------------------------------------------------------------------------------------------------------ head forward
def head_fwd_ref(z, W1, b1, W2, b2, h1):
    """k_head_fwd on its own inputs.  z [B, 2Hp] (workspace code 2), the head parameters of head_params, h1 [B, Hp]
    the kernel's hidden layer (code 1).  -> (pre, pre_bar, pred, pred_bar) in float64.

    pre = W1 z + b1.  Each output is two interleaved chains of Hp FMAs (even / odd k), then a0 + a1 and + b1: a term
    passes through at most Hp + 2 roundings, pre_bar = gamma(Hp + 2) (|W1| |z| + |b1|).  ReLU is 1-Lipschitz, so h1
    must lie within pre_bar of relu(pre) whichever side of 0 a pre-activation within the bar rounds to.

    pred = W2 h1 + b2 on the kernel's own h1 (so the reference follows the kernel's ReLU mask): lane j of the graph's warp
    adds h1[n] W2[n] for n = j, j + 32, ... (ceil(Hp / 32) FMAs, across the W1 slices as well), a 5-step shuffle tree
    adds the lanes and b2 comes last: pred_bar = gamma(ceil(Hp / 32) + 6) (|W2| |h1| + |b2|)."""
    Hp = W1.shape[0]
    z, W1, b1, W2, b2, h1 = (t.double() for t in (z, W1, b1, W2, b2, h1))
    pre = z @ W1.T + b1
    pre_bar = gamma(Hp + 2) * (z.abs() @ W1.abs().T + b1.abs())
    pred = h1 @ W2 + b2
    pred_bar = gamma(math.ceil(Hp / 32) + 6) * (h1.abs() @ W2.abs() + b2.abs())
    return pre, pre_bar, pred, pred_bar


# ------------------------------------------------------------------------------------------------------ head backward
def head_bwd_ref(dg, z, h1, W1, W2, ids, n_entry):
    """k_head_bwd on its own inputs: dg [B] (d_global), z, h1 as the forward left them, W1 / W2 of head_params, ids the
    entry ids.  The ReLU mask is the kernel's (h1 > 0).  -> dict name -> (ref, bar), float64, in the engine's layout:
    dpool [B, Hp], entry [n_entry, Hp], W1 [Hp, 2Hp], b1 [Hp], W2 [Hp], b2 [1].

    dh = dg W2 (h1 > 0) rounds once.  dz = dh W1 is two interleaved chains of Hp / 2 FMAs and their sum, so a term of
    dz passes through 1 + Hp / 2 + 1 roundings: dpool's bar is gamma(Hp / 2 + 2) |dh| |W1|.  A row r of the entry
    gradient adds the entry half of dz of its n_r graphs with n_r atomics (the first into 0, the padded copy's unpack
    add one more): gamma(Hp / 2 + 2 + n_r + 1).

    The weight gradients sum their 8 graphs per CTA (an FMA / addition chain of 8) and add the CTA's sum atomically
    (ceil(B / 8) additions, plus the unpack add at Hp > H): dW1 = dh^T z and db1 = sum dh carry the dh rounding as well,
    gamma(1 + 8 + ceil(B / 8) + 1); dW2 = dg^T h1 gamma(8 + ceil(B / 8) + 1); db2 = sum dg lands in the flat buffer
    directly, gamma(8 + ceil(B / 8))."""
    Hp = W1.shape[0]
    B = dg.numel()
    dg, z, h1, W1, W2 = (t.double() for t in (dg, z, h1, W1, W2))
    ids = torch.as_tensor(ids).long()
    mask = (h1 > 0).double()
    dh = dg[:, None] * W2[None, :] * mask
    dz = dh @ W1
    dz_abs = dh.abs() @ W1.abs()
    n_r = torch.bincount(ids, minlength=n_entry).double()
    ent = torch.zeros(n_entry, Hp, dtype=torch.float64).index_add_(0, ids, dz[:, Hp:])
    ent_abs = torch.zeros(n_entry, Hp, dtype=torch.float64).index_add_(0, ids, dz_abs[:, Hp:])
    g_ent = (n_r + Hp // 2 + 3) * U
    ncta = math.ceil(B / HEAD_G)
    gw = gamma(1 + HEAD_G + ncta + 1)
    return {
        "dpool": (dz[:, :Hp], gamma(Hp // 2 + 2) * dz_abs[:, :Hp]),
        "entry": (ent, (g_ent / (1 - g_ent))[:, None] * ent_abs),
        "W1": (dh.T @ z, gw * (dh.abs().T @ z.abs())),
        "b1": (dh.sum(0), gw * dh.abs().sum(0)),
        "W2": (h1.T @ dg, gamma(HEAD_G + ncta + 1) * (h1.abs().T @ dg.abs())),
        "b2": (dg.sum().reshape(1), gamma(HEAD_G + ncta) * dg.abs().sum().reshape(1)),
    }


# ------------------------------------------------------------------------------------------------------ edge tables
def table_fwd_ref(emb, We):
    """T = emb . We^T (T_if = if_emb WeA^T, T_rpc = rpc_emb WeB^T): one k_small_gemm chain of Hp FMAs per output,
    bar gamma(Hp) |emb| |We|^T."""
    Hp = We.shape[0]
    emb, We = emb.double(), We.double()
    return emb @ We.T, gamma(Hp) * (emb.abs() @ We.abs().T)


def split_k(n):
    """table_grads: the interface half takes split-K 8 from 512 rows, every other problem one pass."""
    return 8 if n >= 512 else 1


def table_wgrad_ref(dT, emb, ks):
    """dWe = dT^T . emb [Hp, Hp] (dWeA from dt_if, dWeB from dt_rpc).  Each of the ks parts is a chain of ceil(n / ks)
    FMAs, added atomically into the zeroed packed gradient (ks additions; at ks = 1 the one addition into 0 is exact):
    bar gamma(ceil(n / ks) + ks) |dT|^T |emb|."""
    n = dT.shape[0]
    dT, emb = dT.double(), emb.double()
    return dT.T @ emb, gamma(math.ceil(n / ks) + ks) * (dT.abs().T @ emb.abs())


def table_dgrad_ref(dTs, Wes):
    """d emb = sum over layers of dT[l] . We[l] [n, Hp]: per layer a chain of Hp FMAs, the L layers added atomically
    (L additions), plus the unpack add of the padded copy at Hp > H: bar gamma(Hp + L + 1) sum_l |dT[l]| |We[l]|."""
    Hp, L = Wes[0].shape[0], len(Wes)
    ref = sum(dT.double() @ We.double() for dT, We in zip(dTs, Wes))
    bar = gamma(Hp + L + 1) * sum(dT.double().abs() @ We.double().abs() for dT, We in zip(dTs, Wes))
    return ref, bar


# ------------------------------------------------------------------------------------------------------ float32 restatements
def fma32(a, b, c):
    """fmaf: the float64 product of two floats is exact, one rounding to float32 after the addition (a double rounding
    through float64 differs from fmaf only by 2^-29 relative, far inside every bar)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def tf32(x):
    """Operands rounded to TF32 (10 mantissa bits, round to nearest) -- what a tensor-core GEMM would read."""
    b = np.asarray(x, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _atomic_sum(parts, rng, start=None):
    """float32 atomic additions of parts[i] (arrays of one shape) into `start` (default 0) in a random order."""
    acc = np.zeros_like(parts[0], np.float32) if start is None else start.astype(np.float32).copy()
    for i in (rng.permutation(len(parts)) if rng is not None else range(len(parts))):
        acc = (acc + parts[i]).astype(np.float32)
    return acc


def head_fwd_f32(z, W1p, b1, W2, b2, defect=None):
    """k_head_fwd in float32.  W1p is the engine's [Hp, 2Hp].  defect: 'slice' stages the rows of the previous slice for
    every slice after the first (ns < Hp only)."""
    z, W1p, b1, W2 = (np.asarray(t, np.float32) for t in (z, W1p, b1, W2))
    B, Hp = z.shape[0], W1p.shape[0]
    ns = fwd_slice(Hp)
    rows = np.arange(Hp)
    if defect == "slice":
        rows = np.where(rows >= ns, rows - ns, rows)
    W = W1p[rows]
    a0 = np.zeros((B, Hp), np.float32)
    a1 = np.zeros((B, Hp), np.float32)
    for k in range(0, 2 * Hp, 2):
        a0 = fma32(z[:, k:k + 1], W[None, :, k], a0)
        a1 = fma32(z[:, k + 1:k + 2], W[None, :, k + 1], a1)
    h1 = np.maximum((a0 + a1) + b1[None, :], F32(0))
    o = np.zeros((B, 32), np.float32)
    for n in range(Hp):
        o[:, n % 32] = fma32(h1[:, n], W2[n], o[:, n % 32])
    lanes = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        o = o + o[:, lanes ^ off]
    return h1, o[:, 0] + F32(np.asarray(b2).reshape(-1)[0])


def head_bwd_f32(dg, z, h1, W1p, W2, ids, n_entry, rng=None, defect=None):
    """k_head_bwd in float32, the atomics of every CTA / graph in a random order (rng).  -> dict like head_bwd_ref.
    defect: 'no_mask' drops the ReLU mask, 'drop_tail' loses the last partial CTA's weight gradients (B % 8 != 0)."""
    dg, z, h1, W1p, W2 = (np.asarray(t, np.float32) for t in (dg, z, h1, W1p, W2))
    ids = np.asarray(ids)
    B, Hp = z.shape[0], W1p.shape[0]
    dh = (dg[:, None] * W2[None, :]).astype(np.float32)
    if defect != "no_mask":
        dh = np.where(h1 > 0, dh, F32(0))
    a0 = np.zeros((B, 2 * Hp), np.float32)
    a1 = np.zeros((B, 2 * Hp), np.float32)
    for n in range(0, Hp, 2):
        a0 = fma32(dh[:, n:n + 1], W1p[None, n], a0)
        a1 = fma32(dh[:, n + 1:n + 2], W1p[None, n + 1], a1)
    dz = a0 + a1
    ent = np.zeros((n_entry, Hp), np.float32)
    for b in (rng.permutation(B) if rng is not None else range(B)):
        ent[ids[b]] = ent[ids[b]] + dz[b, Hp:]
    ncta = -(-B // HEAD_G)
    if defect == "drop_tail" and B % HEAD_G:
        ncta -= 1
    pW1, pb1, pW2, pb2 = [], [], [], []
    for c in range(ncta):
        g = range(c * HEAD_G, min(B, c * HEAD_G + HEAD_G))
        tW1 = np.zeros((Hp, 2 * Hp), np.float32)
        tb1 = np.zeros(Hp, np.float32)
        tW2 = np.zeros(Hp, np.float32)
        tb2 = np.zeros(1, np.float32)
        for b in g:
            tW1 = fma32(dh[b][:, None], z[b][None, :], tW1)
            tb1 = tb1 + dh[b]
            tW2 = fma32(dg[b], h1[b], tW2)
            tb2 = tb2 + dg[b]
        pW1.append(tW1)
        pb1.append(tb1)
        pW2.append(tW2)
        pb2.append(tb2)
    empty = lambda *s: [np.zeros(s, np.float32)]
    return {"dpool": dz[:, :Hp], "entry": ent,
            "W1": _atomic_sum(pW1 or empty(Hp, 2 * Hp), rng), "b1": _atomic_sum(pb1 or empty(Hp), rng),
            "W2": _atomic_sum(pW2 or empty(Hp), rng), "b2": _atomic_sum(pb2 or empty(1), rng)}


def small_gemm_f32(A, Bt, ks=1, rng=None, defect=None):
    """k_small_gemm: C[m, n] = sum_k A[m, k] Bt[n, k], K split in ks parts of ceil(K / ks) rows, each an FMA chain,
    the parts added atomically in a random order (into 0).  defect: 'tf32' rounds both operands to TF32, 'split_floor'
    cuts K into parts of floor(K / ks) rows and so skips the tail rows."""
    A, Bt = np.asarray(A, np.float32), np.asarray(Bt, np.float32)
    if defect == "tf32":
        A, Bt = tf32(A), tf32(Bt)
    K = A.shape[1]
    klen = K // ks if defect == "split_floor" else -(-K // ks)
    parts = []
    for p in range(ks):
        acc = np.zeros((A.shape[0], Bt.shape[0]), np.float32)
        for k in range(p * klen, min(K, p * klen + klen)):
            acc = fma32(A[:, k:k + 1], Bt[None, :, k], acc)
        parts.append(acc)
    return _atomic_sum(parts, rng)


def unpack_f32(G0, packed, defect=None):
    """k_unpack: grads += packed (float32), 'overwrite' stores instead of adding."""
    G0, packed = np.asarray(G0, np.float32), np.asarray(packed, np.float32)
    return packed.copy() if defect == "overwrite" else (G0 + packed).astype(np.float32)
