"""-m gpu tests of the node kernels of csrc/nodeops.cu against float64 references built from the same fp32 inputs, called
through the exported C entries (and through ops / nn where those pad):

  * BatchNorm (+ReLU) forward / backward: pert_bn_fwd, pert_bn_bwd, nn.BatchNorm1d;
  * the local head + probability-weighted add-pool: pert_pool_fwd, pert_pool_bwd, ops.pool_local, nn.global_add_pool;
  * the embedding gather / scatter-add and the X0 concat: pert_embedding_fwd, pert_embedding_bwd, pert_copy_cols,
    ops.embedding, ops.embed_concat.

Every output buffer starts filled with a sentinel (inputs carry NaN in their stride gaps and spare rows), and the
padding columns, stride gaps and rows past N are checked to be untouched.

Two kinds of data:

  * exactly representable data -- small integers, probabilities and node counts that are powers of two -- where every
    sum is exact in fp32 in any order, so a gather or a sum is compared bit for bit whatever the atomic order; and a
    pool of random data over graphs that touch at most two 8-row groups, whose two partial sums commute, so the kernel
    is compared bit for bit with a numpy fp32 restatement of its rounding order;
  * random data under element-wise bars, each derived below from the kernel's arithmetic.  u = 2^-24 (fp32 unit
    roundoff); a sequential fp32 sum of terms t_i over a chain of depth D is off by at most D u sum |t_i| (the standard
    gamma_D bound, D u << 1 throughout); every further rounding adds u times the size of the value it rounds.

BatchNorm forward, training (k_bn_partial + bn_batch_stats).  With rl = 256 / (H/4) row lanes, a thread sums
ceil(128/rl) rows of its 128-row chunk and the rl partials are summed in shared memory: depth Df = ceil(128/rl) + rl.
  * mean: chunk mean mu_b is off by delta_b <= (Df + 1) u mean_b|x| (sum + division); the chunks combine in fp64 and
    the result is rounded to fp32:  |mean - m| <= (Df + 2) u mean|x| + nb 2^-53 mean|x|.
  * variance: q_b = sum (x - mu_b)^2 in fp32 (a rounded difference and an fma per term: (Df + 3) u q_b), and
    S2 - S1^2/N in fp64.  Centring chunk b on mu_b = m_b + delta_b instead of its exact mean m_b moves the variance by
    (2 sum_b n_b (m_b - m) delta_b + 2 sum_b n_b delta_b^2 - ...) / N.  So
    |var - v| <= [(Df + 3) u M2 + 2 sum_b n_b |m_b - m| delta_b + 2 sum_b n_b delta_b^2] / N + (2 nb + 8) 2^-53 mean x^2.
  * rstd = 1/sqrt(var + eps) rounded to fp32: by the mean value theorem
    |rstd - r| <= Evar / 2 (v + eps - Evar)^-3/2 + 2 u r.
  * running statistics, fp32 (1 - mom) rs + mom s with s the batch mean or the unbiased variance v N/(N-1):
    3 u (|(1 - mom) rs| + |mom s|) + mom Es, Es the bar of s (Evar N/(N-1) + u v N/(N-1) for the variance).
  * y = fma((x - mean) rstd, gamma, beta), compared with the fp64 value of the same formula at the kernel's own fp32
    mean / rstd (checked on their own above, so a failure says which part broke): two roundings inside, one in the fma:
    3 u (|gamma| |x - mean| rstd + |y|); ReLU is 1-Lipschitz.  A constant column has x - mean = 0: y is beta exactly.
BatchNorm forward, eval: mean = running_mean exactly; rstd = 1/sqrtf(rv + eps): 3 u r; y as above.

BatchNorm backward (k_bn_bwd_reduce + k_bn_bwd_apply), compared with fp64 at the forward's fp32 mean / rstd:
  g = dy (y > 0 if relu), xh = (x - mean) rstd, a = sum g, b = sum g xh.  A thread sums ceil(64/rl) rows, the rl
  partials are summed in shared memory and ceil(N/64) CTAs add theirs with fp32 atomics:
  depth Db = ceil(64/rl) + rl + ceil(N/64);  Ea = Db u sum|g|,  Eb = (Db + 3) u sum |g xh| (xh: two roundings, fma).
  * dx (training) = gamma rstd (g - a/N - xh b/N): at most 8 roundings on the longest path (1/N, the products and the
    two differences, the two outer products):  |gamma| rstd (8 u (|g| + |a|/N + |xh| |b|/N) + (Ea + |xh| Eb)/N).
  * dx (eval) = gamma rstd g: 3 u |gamma rstd g|.
  * dbeta += a, dgamma += b (accumulated into non-zero buffers): Ea + 2 u (|dbeta0| + |a|), same with b / Eb.

Pool (k_pool_fwd / k_pool_bwd): a group of LPR lanes owns 8 consecutive rows.
  * local = <x, w> + b: a float4 dot per lane, lane partials summed by shuffles: (H + 2) u (sum |x w| + |b|).
  * dx = fma(dlocal, w, (p / n) dpool[batch]): three roundings: 3 u (|dpool p / n| + |dlocal w|).
  * dw_local += sum dlocal x, db_local += sum dlocal: 8 rows per lane, 256/LPR groups per CTA into shared memory, one
    atomic per CTA: depth 8 + 256/LPR + n_cta + 1 on sum |dlocal x| (sum |dlocal|), plus 2 u of the start value.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
U64 = 2.0 ** -53
SENT = 12345.0
BADARG, RANGE = -1, -3
BN_ROWS, BN_BWD_ROWS, POOL_ROWS, EB_RUN = 128, 64, 8, 8
EPS = float(np.float32(1e-5))
POOL_WIDTHS = [4, 8, 16, 32, 64, 96, 128, 192, 256]
LPR = {4: 1, 8: 2, 16: 4, 32: 8, 64: 16, 96: 8, 128: 32, 192: 16, 256: 32}   # dispatch_h: lanes per row


def _L():
    from pert_gnn_kdd23_b200 import _lib

    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _f32(v):
    return float(np.float32(v))


def _strided(data, ld, extra_rows=2, fill=float("nan")):
    """[N, H] data in a [N + extra_rows, ld] buffer whose stride gap and spare rows hold `fill`."""
    N, H = data.shape
    buf = torch.full((N + extra_rows, ld), fill, device="cuda", dtype=torch.float32)
    buf[:N, :H] = data
    return buf


def _untouched(buf, N, H, what):
    """Columns >= H and rows >= N of a sentinel-filled output buffer were not written."""
    assert bool((buf[:N, H:] == SENT).all()), f"{what}: stride gap written"
    assert bool((buf[N:] == SENT).all()), f"{what}: rows past N written"


def _ratio(got, ref, bar):
    err = (got.double() - ref).abs()
    return float((err / bar).max()) if err.numel() else 0.0


def _assert_bar(got, ref, bar, what):
    r = _ratio(got, ref, bar)
    assert r <= 1.0, f"{what}: element-wise error {r:.3g} x the bar"


# ==================================================================================================== BatchNorm
def _bn_state(H, g, mom=0.1):
    return dict(gamma=(1 + 0.3 * torch.randn(H, generator=g)).cuda(), beta=(0.2 * torch.randn(H, generator=g)).cuda(),
                rm=(0.1 * torch.randn(H, generator=g)).cuda(), rv=(1 + torch.rand(H, generator=g)).cuda(),
                nbt=torch.tensor([3], dtype=torch.int64).cuda(), mom=mom)


def _bn_fwd(xbuf, N, H, s, training, relu, ld_y):
    L = _L()
    y = torch.full((N + 2, ld_y), SENT, device="cuda")
    mean = torch.full((H + 4,), SENT, device="cuda")
    rstd = torch.full((H + 4,), SENT, device="cuda")
    wsb = L.pert_bn_workspace_bytes(N, H)
    ws = torch.full((wsb // 8 + 1,), float("nan"), device="cuda", dtype=torch.float64)
    rc = L.pert_bn_fwd(xbuf.data_ptr(), xbuf.stride(0), s["gamma"].data_ptr(), s["beta"].data_ptr(), s["rm"].data_ptr(),
                       s["rv"].data_ptr(), s["nbt"].data_ptr(), EPS, s["mom"], int(training), int(relu),
                       mean.data_ptr(), rstd.data_ptr(), y.data_ptr(), ld_y, N, H, ws.data_ptr(), wsb, _st())
    torch.cuda.synchronize()
    return rc, y, mean, rstd


def _bn_bwd(dybuf, y, xbuf, mean, rstd, s, relu, training, N, H, ld_dx, dg0, db0):
    L = _L()
    dx = torch.full((N + 2, ld_dx), SENT, device="cuda")
    dgamma = torch.cat([dg0, torch.full((4,), SENT, device="cuda")])
    dbeta = torch.cat([db0, torch.full((4,), SENT, device="cuda")])
    sums = torch.full((2 * H,), float("nan"), device="cuda")
    rc = L.pert_bn_bwd(dybuf.data_ptr(), dybuf.stride(0), y.data_ptr(), y.stride(0), xbuf.data_ptr(), xbuf.stride(0),
                       mean.data_ptr(), rstd.data_ptr(), s["gamma"].data_ptr(), int(relu), int(training),
                       dx.data_ptr(), ld_dx, dgamma.data_ptr(), dbeta.data_ptr(), sums.data_ptr(), N, H, _st())
    torch.cuda.synchronize()
    return rc, dx, dgamma, dbeta


def _bn_fwd_ref(x64, H):
    """fp64 batch mean / biased variance and the bars on the kernel's mean and variance (module docstring)."""
    N = x64.size(0)
    rl = 256 // (H // 4)
    Df = math.ceil(BN_ROWS / rl) + rl
    m = x64.mean(0)
    M2 = ((x64 - m) ** 2).sum(0)
    v = M2 / N
    nb = math.ceil(N / BN_ROWS)
    pad = nb * BN_ROWS - N
    xp = torch.nn.functional.pad(x64, (0, 0, 0, pad)).view(nb, BN_ROWS, H)
    n_b = torch.full((nb, 1), float(BN_ROWS), device=x64.device, dtype=torch.float64)
    n_b[-1] = BN_ROWS - pad
    m_b = xp.sum(1) / n_b
    delta_b = (Df + 1) * U * xp.abs().sum(1) / n_b
    absm = x64.abs().mean(0)
    Em = (Df + 2) * U * absm + nb * U64 * absm
    Evar = ((Df + 3) * U * M2 + (2 * n_b * (m_b - m).abs() * delta_b).sum(0) + (2 * n_b * delta_b ** 2).sum(0)) / N \
        + (2 * nb + 8) * U64 * (x64 * x64).mean(0)
    return m, v, Em, Evar


def _check_bn_fwd(x64, N, H, s0, s, y, mean, rstd, training, relu, tag):
    m_k, rs_k = mean[:H].double(), rstd[:H].double()
    assert bool((mean[H:] == SENT).all()) and bool((rstd[H:] == SENT).all()), f"mean / rstd past H written ({tag})"
    mom = _f32(s0["mom"])
    if training:
        m, v, Em, Evar = _bn_fwd_ref(x64, H)
        _assert_bar(mean[:H], m, Em, f"mean ({tag})")
        r = 1.0 / torch.sqrt(v + EPS)
        Ers = 0.5 * Evar * (v + EPS - Evar).clamp_min(EPS) ** -1.5 + 2 * U * r
        _assert_bar(rstd[:H], r, Ers, f"rstd ({tag})")
        rm0, rv0 = s0["rm"].double(), s0["rv"].double()
        rm_ref = (1 - mom) * rm0 + mom * m
        _assert_bar(s["rm"], rm_ref, 3 * U * ((1 - mom) * rm0.abs() + mom * m.abs()) + mom * Em, f"running_mean ({tag})")
        k = N / (N - 1) if N > 1 else 1.0
        unb = v * k
        rv_ref = (1 - mom) * rv0 + mom * unb
        _assert_bar(s["rv"], rv_ref, 3 * U * ((1 - mom) * rv0.abs() + mom * unb) + mom * (Evar * k + U * unb),
                    f"running_var ({tag})")
        assert int(s["nbt"]) == int(s0["nbt"]) + 1, f"num_batches_tracked ({tag})"
    else:
        assert torch.equal(mean[:H], s0["rm"]), f"eval mean is the running mean ({tag})"
        r = 1.0 / torch.sqrt(s0["rv"].double() + EPS)
        _assert_bar(rstd[:H], r, 3 * U * r, f"eval rstd ({tag})")
        for k in ("rm", "rv", "nbt"):
            assert torch.equal(s[k], s0[k]), f"eval changed {k} ({tag})"
    ga, be = s0["gamma"].double(), s0["beta"].double()
    d = x64 - m_k
    y_ref = d * rs_k * ga + be
    bar = 3 * U * (ga.abs() * d.abs() * rs_k + y_ref.abs())
    if relu:
        y_ref = y_ref.clamp_min(0)
    # a zero bar (x == mean, beta == 0) asks for equality
    _assert_bar(y[:N, :H], y_ref, bar.clamp_min(1e-300), f"y ({tag})")
    _untouched(y, N, H, f"y ({tag})")


def _check_bn_bwd(x64, dy64, y, mean, rstd, s0, relu, training, N, H, dx, dgamma, dbeta, dg0, db0, tag):
    m_k, rs_k, ga = mean[:H].double(), rstd[:H].double(), s0["gamma"].double()
    g = dy64 * (y[:N, :H] > 0).double() if relu else dy64
    xh = (x64 - m_k) * rs_k
    a, b = g.sum(0), (g * xh).sum(0)
    rl = 256 // (H // 4)
    Db = math.ceil(BN_BWD_ROWS / rl) + rl + math.ceil(N / BN_BWD_ROWS)
    Ea = Db * U * g.abs().sum(0)
    Eb = (Db + 3) * U * (g * xh).abs().sum(0)
    if training:
        dx_ref = ga * rs_k * (g - a / N - xh * b / N)
        bar = ga.abs() * rs_k * (8 * U * (g.abs() + a.abs() / N + xh.abs() * b.abs() / N) + (Ea + xh.abs() * Eb) / N)
    else:
        dx_ref = ga * rs_k * g
        bar = 3 * U * (ga * rs_k * g).abs()
    _assert_bar(dx[:N, :H], dx_ref, bar.clamp_min(1e-300), f"dx ({tag})")
    _untouched(dx, N, H, f"dx ({tag})")
    assert bool(torch.isfinite(dx[:N, :H]).all()), f"dx not finite ({tag})"
    dg0d, db0d = dg0.double(), db0.double()
    _assert_bar(dbeta[:H], db0d + a, Ea + 2 * U * (db0d.abs() + a.abs()) + 1e-300, f"dbeta += ({tag})")
    _assert_bar(dgamma[:H], dg0d + b, Eb + 2 * U * (dg0d.abs() + b.abs()) + 1e-300, f"dgamma += ({tag})")
    assert bool((dgamma[H:] == SENT).all()) and bool((dbeta[H:] == SENT).all()), f"dgamma / dbeta past H ({tag})"


def _bn_case(N, H, training, relu, seed, ld_x=None, ld_y=None, ld_dy=None, ld_dx=None, x=None, dy=None, mom=0.1):
    """One forward + backward through the C entries, every output checked against fp64."""
    g = torch.Generator().manual_seed(seed)
    if x is None:
        x = (2.0 * torch.randn(N, H, generator=g) + 0.5).cuda()
    if dy is None:
        dy = torch.randn(N, H, generator=g).cuda()
    ld_x, ld_y, ld_dy, ld_dx = ld_x or H, ld_y or H, ld_dy or H, ld_dx or H
    s0 = _bn_state(H, g, mom)
    s = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in s0.items()}
    xbuf, dybuf = _strided(x, ld_x), _strided(dy, ld_dy)
    tag = f"N={N} H={H} train={training} relu={relu}"
    rc, y, mean, rstd = _bn_fwd(xbuf, N, H, s, training, relu, ld_y)
    assert rc == 0, f"pert_bn_fwd rc={rc} ({tag})"
    x64 = x.double()
    _check_bn_fwd(x64, N, H, s0, s, y, mean, rstd, training, relu, tag)
    dg0 = torch.randn(H, generator=g).cuda()
    db0 = torch.randn(H, generator=g).cuda()
    rc, dx, dgamma, dbeta = _bn_bwd(dybuf, y, xbuf, mean, rstd, s0, relu, training, N, H, ld_dx, dg0, db0)
    assert rc == 0, f"pert_bn_bwd rc={rc} ({tag})"
    _check_bn_bwd(x64, dy.double(), y, mean, rstd, s0, relu, training, N, H, dx, dgamma, dbeta, dg0, db0, tag)
    return y, mean, s0


@pytest.mark.parametrize("H", list(range(4, 1025, 4)))
def test_bn_every_width(H):
    """Every width the entries accept, at N = 129 (one full 128-row chunk and a one-row tail): training, and eval with
    the other ReLU setting."""
    relu = H % 8 == 0
    _bn_case(129, H, True, relu, seed=H)
    _bn_case(129, H, False, not relu, seed=H + 1)


@pytest.mark.parametrize("H", [12, 1024])
@pytest.mark.parametrize("N", [2, 3, 63, 64, 65, 127, 128, 129, 4097])
def test_bn_row_counts(N, H):
    """Row counts around the 128-row forward and 64-row backward chunks, at a narrow width (21 row lanes, so the 8-row
    unroll ends in a partial step) and the widest (one row lane)."""
    _bn_case(N, H, True, True, seed=N * 7 + H)
    _bn_case(N, H, False, False, seed=N * 7 + H + 1)


@pytest.mark.parametrize("H", [64, 100, 512])
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("relu", [True, False])
def test_bn_strided_layouts(H, training, relu):
    """Row strides above H on every operand; dx at ld = H + 16 as the engine writes it into the next layer's input."""
    _bn_case(1000, H, training, relu, seed=H + 10 * training + relu, ld_x=H + 8, ld_y=H + 4, ld_dy=2 * H,
             ld_dx=H + 16, mom=0.3)


@pytest.mark.parametrize("H", [64, 260])
def test_bn_stress_columns(H):
    """A column of mean 1e3 / std 1, a constant column, a column with one outlier; the upstream gradient has a common
    offset (1 + 0.01 randn), so the mean terms cancel most of dz."""
    N = 4097
    g = torch.Generator().manual_seed(H)
    x = torch.randn(N, H, generator=g)
    x[:, 0] = 1000.0 + torch.randn(N, generator=g)
    x[:, 1] = 7.25
    x[N // 3, 2] = 1e4
    dy = 1.0 + 0.01 * torch.randn(N, H, generator=g)
    for training, relu in ((True, False), (True, True), (False, False)):
        y, mean, s0 = _bn_case(N, H, training, relu, seed=H, x=x.cuda(), dy=dy.cuda())
        if training:
            assert float(mean[1]) == 7.25
            beta1 = float(s0["beta"][1])
            col = y[:N, 1]
            want = max(beta1, 0.0) if relu else beta1
            assert bool((col == want).all()), "a constant column must give y = beta exactly"


@pytest.mark.parametrize("H", [4, 64, 256])
def test_bn_large_batch(H):
    """About 1e6 rows: 7813 fp64-atomic chunks forward, 15626 fp32-atomic chunks backward, shifted gradient."""
    N = 1_000_037
    g = torch.Generator(device="cuda").manual_seed(H)
    x = 3.0 * torch.randn(N, H, generator=g, device="cuda") + 5.0
    dy = 1.0 + 0.01 * torch.randn(N, H, generator=g, device="cuda")
    _bn_case(N, H, True, H != 64, seed=H, x=x, dy=dy)


@pytest.mark.parametrize("H", [260, 512, 1024])
def test_bn_wide_training_updates_running_stats(H):
    """Training above H = 256 (k_bn_partial used to be launched with more threads than its launch bound allows, after the
    workspace was zeroed, so the apply stored mean 0 / variance 0 into the running statistics before the error came
    back): the call succeeds and the running statistics are the fp64 update.  A call the entry refuses leaves them
    alone."""
    _bn_case(4097, H, True, False, seed=H)
    g = torch.Generator().manual_seed(H)
    s0 = _bn_state(H, g)
    s = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in s0.items()}
    xbuf = _strided(torch.randn(300, H + 4, generator=g).cuda(), H + 4)
    rc, y, mean, rstd = _bn_fwd(xbuf, 300, H + 4 if H == 1024 else H + 2, s, True, False, H + 4)
    assert rc == BADARG
    for k in ("rm", "rv", "nbt"):
        assert torch.equal(s[k], s0[k]), f"a refused call changed {k}"
    assert bool((y == SENT).all()) and bool((mean == SENT).all())


def test_bn_rejects_width_1028():
    g = torch.Generator().manual_seed(0)
    H = 1028
    s0 = _bn_state(H, g)
    s = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in s0.items()}
    xbuf = _strided(torch.randn(129, H, generator=g).cuda(), H)
    for training in (1, 0):
        rc, y, _, _ = _bn_fwd(xbuf, 129, H, s, training, 0, H)
        assert rc == BADARG and bool((y == SENT).all())
    assert all(torch.equal(s[k], s0[k]) for k in ("rm", "rv", "nbt"))


# ---------------------------------------------------------------------------------------------------- nn shim
def _padded_reference(x, dy, H, affine, training, relu, mod):
    """The C entries on the zero-padded [N, round4(H)] problem: what the shim must reproduce bit for bit (N = 64 is one
    forward and one backward chunk, so neither has an atomic-order freedom)."""
    N, H4 = x.size(0), (H + 3) // 4 * 4
    pad = lambda t, v=0.0: torch.nn.functional.pad(t, (0, H4 - H), value=v)  # noqa: E731
    s = dict(gamma=pad(mod.weight.detach()) if affine else torch.ones(H4, device="cuda"),
             beta=pad(mod.bias.detach()) if affine else torch.zeros(H4, device="cuda"),
             rm=pad(mod.running_mean.clone()), rv=pad(mod.running_var.clone(), 1.0),
             nbt=mod.num_batches_tracked.clone(), mom=mod.momentum)
    xbuf = _strided(pad(x), H4, extra_rows=0)
    rc, y, mean, rstd = _bn_fwd(xbuf, N, H4, s, training, relu, H4)
    assert rc == 0
    rc, dx, dgamma, dbeta = _bn_bwd(_strided(pad(dy), H4, extra_rows=0), y[:N], xbuf, mean, rstd, s, relu, training,
                                    N, H4, H4, torch.zeros(H4, device="cuda"), torch.zeros(H4, device="cuda"))
    assert rc == 0
    return y[:N, :H], dx[:N, :H], dgamma[:H], dbeta[:H], s


@pytest.mark.parametrize("H", list(range(1, 21)) + [255, 257, 300, 1021])
def test_batchnorm_shim_pads_to_whole_float4s(H):
    """nn.BatchNorm1d at any width: bit-identical to the C entries on the zero-padded problem (whose arithmetic the
    tests above check against fp64), padding dropped from every output, running statistics of the real columns only."""
    from pert_gnn_kdd23_b200.nn import BatchNorm1d

    N = 64
    torch.manual_seed(H)
    for training, relu, affine in ((True, True, True), (False, False, True), (True, False, False)):
        mod = BatchNorm1d(H, affine=affine).cuda()
        if affine:
            with torch.no_grad():
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-1, 1)
        mod.running_mean.normal_()
        mod.running_var.uniform_(0.5, 2)
        mod.train(training)
        x = (torch.randn(N, H) * 2 + 1).cuda()
        dy = torch.randn(N, H).cuda()
        y_ref, dx_ref, dg_ref, db_ref, s = _padded_reference(x, dy, H, affine, training, relu, mod)
        xr = x.clone().requires_grad_()
        y = mod(xr, relu=relu)
        y.backward(dy)
        tag = f"H={H} train={training} relu={relu} affine={affine}"
        assert y.shape == (N, H) and torch.equal(y, y_ref), f"y ({tag})"
        assert torch.equal(xr.grad, dx_ref), f"dx ({tag})"
        if affine:
            assert torch.equal(mod.weight.grad, dg_ref) and torch.equal(mod.bias.grad, db_ref), f"dgamma / dbeta ({tag})"
        else:
            assert mod.weight is None and mod.bias is None
        assert torch.equal(mod.running_mean, s["rm"][:H]) and torch.equal(mod.running_var, s["rv"][:H]), tag
        assert int(mod.num_batches_tracked) == (1 if training else 0), tag


def test_batchnorm_shim_wide_training_matches_torch():
    """BatchNorm1d(512) in training (it used to raise after corrupting its running statistics): the running statistics
    after two steps equal torch's fp64 module under the forward bars."""
    from pert_gnn_kdd23_b200.nn import BatchNorm1d

    H, N, mom = 512, 300, _f32(0.1)
    torch.manual_seed(0)
    ref = torch.nn.BatchNorm1d(H, momentum=mom).double()
    mod = BatchNorm1d(H).cuda()
    tol_m = tol_v = torch.zeros(H, dtype=torch.float64, device="cuda")
    for step in range(2):       # a step's bar (see _check_bn_fwd) plus the previous bar scaled by (1 - mom)
        x = torch.randn(N, H) * 2 + 1
        rm0, rv0 = ref.running_mean.cuda(), ref.running_var.cuda()
        m, v, Em, Evar = _bn_fwd_ref(x.double().cuda(), H)
        unb = v * N / (N - 1)
        ref(x.double())
        mod(x.cuda())
        tol_m = (1 - mom) * tol_m + 3 * U * ((1 - mom) * rm0.abs() + mom * m.abs()) + mom * Em
        tol_v = (1 - mom) * tol_v + 3 * U * ((1 - mom) * rv0.abs() + mom * unb) + mom * (Evar * N / (N - 1) + U * unb)
    assert int(mod.num_batches_tracked) == 2
    _assert_bar(mod.running_mean, ref.running_mean.cuda(), tol_m, "running_mean")
    _assert_bar(mod.running_var, ref.running_var.cuda(), tol_v, "running_var")


# ==================================================================================================== pool
def _pool_fwd(xbuf, probs, pnn, batch, w, b, N, B, H, with_local=True):
    L = _L()
    pool = torch.full((B + 2, H), SENT, device="cuda")
    local = torch.full((N + 2,), SENT, device="cuda") if with_local else None
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc = L.pert_pool_fwd(xbuf.data_ptr(), xbuf.stride(0), probs.data_ptr(), pnn.data_ptr(), batch.data_ptr(),
                         w.data_ptr() if w is not None else None, b.data_ptr() if b is not None else None,
                         local.data_ptr() if local is not None else None, pool.data_ptr(), N, B, H,
                         status.data_ptr(), _st())
    torch.cuda.synchronize()
    return rc, pool, local, int(status)


def _pool_bwd(dpool, dlocal, xbuf, probs, pnn, batch, w, N, B, H, ld_dx, dw0, db0):
    L = _L()
    dx = torch.full((N + 2, ld_dx), SENT, device="cuda")
    dw = torch.cat([dw0, torch.full((4,), SENT, device="cuda")])
    db = torch.cat([db0, torch.full((3,), SENT, device="cuda")])
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    rc = L.pert_pool_bwd(p(dpool), p(dlocal), xbuf.data_ptr(), xbuf.stride(0), probs.data_ptr(), pnn.data_ptr(),
                         batch.data_ptr(), p(w), dx.data_ptr(), ld_dx, dw.data_ptr(), db.data_ptr(), N, B, H, _st())
    torch.cuda.synchronize()
    return rc, dx, dw, db


def _pool_ref(x64, probs, pnn, batch, w, b, B):
    p, n = probs.double(), pnn.double()
    ok = (batch >= 0) & (batch < B)
    pool = torch.zeros(B, x64.size(1), device="cuda", dtype=torch.float64)
    pool.index_add_(0, batch[ok], (x64 * p[:, None] / n[:, None])[ok])
    local = x64 @ w.double() + b.double() if w is not None else None
    return pool, local


def _pool_bwd_ref(x64, probs, pnn, batch, w, dpool, dlocal, B, dw0, db0):
    p, n = probs.double(), pnn.double()
    ok = ((batch >= 0) & (batch < B)).double()[:, None]
    dx = torch.zeros_like(x64)
    if dpool is not None and B > 0:
        dx += dpool.double()[batch.clamp(0, max(B - 1, 0))] * (p / n)[:, None] * ok
    dw = db = None
    if dlocal is not None:
        dx += dlocal.double()[:, None] * w.double()[None, :]
        dw = dw0.double() + (dlocal.double()[:, None] * x64).sum(0)
        db = db0.double() + dlocal.double().sum()
    return dx, dw, db


def _graph_layout(sizes, skip_every=0):
    """batch ids of consecutive graphs of the given sizes; skip_every > 0 leaves every skip_every-th id empty."""
    ids, gid = [], 0
    for i, sz in enumerate(sizes):
        if skip_every and i % skip_every == skip_every - 1:
            gid += 1
        ids += [gid] * sz
        gid += 1
    return torch.tensor(ids, dtype=torch.int64), gid


def _exact_pool_inputs(batch, B, H, g, xr=4):
    """Integers for x / w / b / gradients, probabilities in {1/4, 1/2, 1, 2} and node counts in {1, 2, 4, 8, 16}: every
    product, quotient and sum below is exact in fp32."""
    N = batch.numel()
    x = torch.randint(-xr, xr + 1, (N, H), generator=g).float()
    probs = 2.0 ** torch.randint(-2, 2, (N,), generator=g).float()
    pnn = 2.0 ** torch.randint(0, 5, (N,), generator=g).float()
    w = torch.randint(-3, 4, (H,), generator=g).float()
    b = torch.randint(-3, 4, (1,), generator=g).float()
    dpool = torch.randint(-4, 5, (B, H), generator=g).float()
    dlocal = torch.randint(-2, 3, (N,), generator=g).float()
    return [t.cuda() for t in (x, probs, pnn, w, b, dpool, dlocal)]


def _pool_exact_case(batch, B, H, seed, ld=None, ld_dx=None, local=True, dpool_on=True, dlocal_on=True, xr=4,
                     expect_status=0):
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    batch = batch.cuda()
    x, probs, pnn, w, b, dpool, dlocal = _exact_pool_inputs(batch, B, H, g, xr)
    ld, ld_dx = ld or H, ld_dx or H
    xbuf = _strided(x, ld)
    tag = f"H={H} N={N} B={B} local={local}"
    rc, pool, loc, status = _pool_fwd(xbuf, probs, pnn, batch, w if local else None, b if local else None, N, B, H,
                                      with_local=local)
    assert rc == 0 and status == expect_status, (rc, status, tag)
    pool_ref, local_ref = _pool_ref(x.double(), probs, pnn, batch, w if local else None, b, B)
    assert torch.equal(pool[:B].double(), pool_ref), f"pool ({tag})"
    assert bool((pool[B:] == SENT).all()), f"pool rows past B ({tag})"
    if local:
        assert torch.equal(loc[:N].double(), local_ref), f"local ({tag})"
        assert bool((loc[N:] == SENT).all()), f"local past N ({tag})"
    dw0 = torch.randint(-5, 6, (H,), generator=g).float().cuda()
    db0 = torch.tensor([3.0], device="cuda")
    dp, dl = (dpool if dpool_on else None), (dlocal if dlocal_on else None)
    rc, dx, dw, db = _pool_bwd(dp, dl, xbuf, probs, pnn, batch, w if dl is not None else None, N, B, H, ld_dx, dw0, db0)
    assert rc == 0, (rc, tag)
    dx_ref, dw_ref, db_ref = _pool_bwd_ref(x.double(), probs, pnn, batch, w, dp, dl, B, dw0, db0)
    assert torch.equal(dx[:N, :H].double(), dx_ref), f"dx ({tag})"
    _untouched(dx, N, H, f"dx ({tag})")
    if dl is not None:
        assert torch.equal(dw[:H].double(), dw_ref) and float(db[0]) == float(db_ref), f"dw / db ({tag})"
    else:
        assert torch.equal(dw[:H], dw0) and float(db[0]) == 3.0, f"dw / db without dlocal ({tag})"
    assert bool((dw[H:] == SENT).all()) and bool((db[1:] == SENT).all())


@pytest.mark.parametrize("H", POOL_WIDTHS)
@pytest.mark.parametrize("local", [True, False])
def test_pool_every_width_exact(H, local):
    """Graphs of 1, 7, 8, 9, 16 and 3 nodes, repeated across the 8-row groups, with empty graph ids in between; strided
    x and dx.  Exact data: pool, local, dx, dw_local, db_local bit for bit."""
    batch, B = _graph_layout([1, 7, 8, 9, 16, 3] * 9 + [9, 1], skip_every=4)
    _pool_exact_case(batch, B + 2, H, seed=H + local, ld=H + 4, ld_dx=H + 8, local=local)


@pytest.mark.parametrize("H", [8, 96, 256])
def test_pool_without_dpool_or_dlocal(H):
    batch, B = _graph_layout([1, 7, 8, 9] * 5)
    _pool_exact_case(batch, B, H, seed=H, dpool_on=False)
    _pool_exact_case(batch, B, H, seed=H, dlocal_on=False)
    _pool_exact_case(batch, B, H, seed=H, dpool_on=False, dlocal_on=False)


@pytest.mark.parametrize("H", [16, 192])
def test_pool_unsorted_batch_and_bad_ids(H):
    """An unsorted batch (runs of all lengths, ids revisited); then out-of-range ids (negative and >= B) set the status
    word and contribute to no pool row or pool gradient."""
    g = torch.Generator().manual_seed(H)
    B = 37
    batch = torch.randint(0, B, (3001,), generator=g)
    batch[100:140] = 5
    _pool_exact_case(batch, B, H, seed=H)
    bad = batch.clone()
    bad[7], bad[8], bad[500], bad[3000] = -1, B, B + 100, -7
    _pool_exact_case(bad, B, H, seed=H, expect_status=RANGE)


@pytest.mark.parametrize("H", [4, 64, 256])
def test_pool_hot_graph(H):
    """One graph of 2^20 nodes between two small ones: 131072 groups add into one pool row (x in {-2..2}, 1/n = 2^-20:
    still exact)."""
    sizes = [5, 1 << 20, 11]
    batch, B = _graph_layout(sizes)
    g = torch.Generator().manual_seed(H)
    N = batch.numel()
    x = torch.randint(-2, 3, (N, H), generator=g).float().cuda()
    probs = torch.ones(N, device="cuda")
    pnn = torch.cat([torch.full((s,), float(s)) for s in sizes]).cuda()
    pnn[:5], pnn[-11:] = 4.0, 8.0
    w = torch.randint(-1, 2, (H,), generator=g).float().cuda()
    b = torch.ones(1, device="cuda")
    batch = batch.cuda()
    rc, pool, loc, status = _pool_fwd(_strided(x, H), probs, pnn, batch, w, b, N, B, H)
    assert rc == 0 and status == 0
    pool_ref, local_ref = _pool_ref(x.double(), probs, pnn, batch, w, b, B)
    assert torch.equal(pool[:B].double(), pool_ref) and torch.equal(loc[:N].double(), local_ref)
    dlocal = torch.randint(-1, 2, (N,), generator=g).float().cuda()
    dpool = torch.randint(-4, 5, (B, H), generator=g).float().cuda()
    z = torch.zeros(H, device="cuda")
    rc, dx, dw, db = _pool_bwd(dpool, dlocal, _strided(x, H), probs, pnn, batch, w, N, B, H, H, z, z[:1])
    dx_ref, dw_ref, db_ref = _pool_bwd_ref(x.double(), probs, pnn, batch, w, dpool, dlocal, B, z, z[:1])
    assert rc == 0 and torch.equal(dx[:N].double(), dx_ref)
    assert torch.equal(dw[:H].double(), dw_ref) and float(db[0]) == float(db_ref)


def _pool_fp32_restatement(x, probs, pnn, batch, B):
    """numpy fp32 restatement of k_pool_fwd's pool: per 8-row group, each run of one graph id summed in row order from
    0 (the terms (x p) / n, two roundings), the run sums added to the zeroed row; valid when every graph touches at most
    two groups (two partial sums commute)."""
    x, p, n, bt = x.cpu().numpy(), probs.cpu().numpy(), pnn.cpu().numpy(), batch.cpu().numpy()
    t = (x * p[:, None]) / n[:, None]
    assert t.dtype == np.float32
    first, last = np.full(B, len(bt)), np.zeros(B, np.int64)
    np.minimum.at(first, bt, np.arange(len(bt)))
    np.maximum.at(last, bt, np.arange(len(bt)))
    assert (last // POOL_ROWS - first // POOL_ROWS).max() <= 1, "a graph touches more than two 8-row groups"
    pool = np.zeros((B, x.shape[1]), np.float32)
    for r0 in range(0, len(bt), POOL_ROWS):
        cur, acc = -1, None
        for r in range(r0, min(r0 + POOL_ROWS, len(bt))):
            if bt[r] != cur:
                if cur >= 0:
                    pool[cur] += acc
                cur, acc = bt[r], np.zeros(x.shape[1], np.float32)
            acc = acc + t[r]
        if cur >= 0:
            pool[cur] += acc
    return pool


@pytest.mark.parametrize("H", POOL_WIDTHS)
def test_pool_random_data(H):
    """Random x, probabilities and node counts: the pool bit for bit against the fp32 restatement of the kernel's
    rounding order ((x p) / n, run sums per 8-row group), local / dx / dw_local / db_local under the module's bars."""
    sizes = [1, 7, 8, 9, 3, 5, 2, 6, 8, 8, 1, 1, 1, 9] * 4
    batch, B = _graph_layout(sizes)
    N = batch.numel()
    g = torch.Generator().manual_seed(H)
    x = torch.randn(N, H, generator=g).cuda()
    probs = torch.rand(N, generator=g).cuda() + 0.05
    pnn = torch.cat([torch.full((s,), float(s)) for s in sizes]).cuda()
    w = torch.randn(H, generator=g).cuda()
    b = torch.randn(1, generator=g).cuda()
    batch = batch.cuda()
    xbuf = _strided(x, H + 4)
    rc, pool, loc, status = _pool_fwd(xbuf, probs, pnn, batch, w, b, N, B, H)
    assert rc == 0 and status == 0
    want = _pool_fp32_restatement(x, probs, pnn, batch, B)
    got = pool[:B].cpu().numpy()
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"pool differs from the fp32 restatement at {len(bad)} elements, first {bad[:4].tolist()}")
    x64 = x.double()
    _, local_ref = _pool_ref(x64, probs, pnn, batch, w, b, B)
    _assert_bar(loc[:N], local_ref, (H + 2) * U * ((x64.abs() @ w.double().abs()) + b.double().abs()), "local")
    dpool = torch.randn(B, H, generator=g).cuda()
    dlocal = torch.randn(N, generator=g).cuda()
    dw0, db0 = torch.randn(H, generator=g).cuda(), torch.randn(1, generator=g).cuda()
    rc, dx, dw, db = _pool_bwd(dpool, dlocal, xbuf, probs, pnn, batch, w, N, B, H, H, dw0, db0)
    assert rc == 0
    dx_ref, dw_ref, db_ref = _pool_bwd_ref(x64, probs, pnn, batch, w, dpool, dlocal, B, dw0, db0)
    sc = (probs.double() / pnn.double())[:, None]
    _assert_bar(dx[:N, :H], dx_ref, 3 * U * (dpool.double()[batch].abs() * sc + (dlocal.double()[:, None] *
                                                                                   w.double()).abs()), "dx")
    groups = math.ceil(N / POOL_ROWS)
    n_cta = math.ceil(groups * LPR[H] / 256)
    D = POOL_ROWS + 256 // LPR[H] + n_cta + 1
    dl64 = dlocal.double()
    _assert_bar(dw[:H], dw_ref, D * U * (dl64[:, None] * x64).abs().sum(0) + 2 * U * dw0.double().abs(), "dw_local")
    _assert_bar(db[:1], db_ref.reshape(1), D * U * dl64.abs().sum() + 2 * U * db0.double().abs(), "db_local")


def test_pool_empty_batch_and_no_graphs():
    """N = 0: the pool is zero-filled and nothing else runs; B = 0: every id is out of range."""
    H = 64
    z = torch.zeros(0, device="cuda")
    zi = torch.zeros(0, dtype=torch.int64, device="cuda")
    rc, pool, _, status = _pool_fwd(torch.zeros(0, H, device="cuda"), z, z, zi, None, None, 0, 3, H, with_local=False)
    assert rc == 0 and status == 0 and bool((pool[:3] == 0).all()) and bool((pool[3:] == SENT).all())
    batch, _ = _graph_layout([3, 5])
    _pool_exact_case(batch, 0, H, seed=1, expect_status=RANGE)
    from pert_gnn_kdd23_b200 import nn, ops

    x = torch.zeros(0, 5, device="cuda", requires_grad=True)
    pool, local = ops.pool_local(x, z, z, zi, None, None, 2)
    assert pool.shape == (2, 5) and bool((pool == 0).all()) and local.shape == (0, 1)
    assert nn.global_add_pool(torch.zeros(0, 5, device="cuda"), zi).shape == (0, 5)


@pytest.mark.parametrize("H", [1, 5, 48, 100, 200])
def test_pool_ops_widths_without_kernel(H):
    """ops.pool_local at widths the kernel lacks (run zero-padded to the next pool width): exact data, the padding leaks
    into no output and no gradient."""
    from pert_gnn_kdd23_b200 import ops

    batch, B = _graph_layout([1, 7, 8, 9, 2] * 6)
    g = torch.Generator().manual_seed(H)
    x, probs, pnn, w, b, dpool, dlocal = _exact_pool_inputs(batch, B, H, g)
    batch = batch.cuda()
    xr, wr, br = (t.clone().requires_grad_() for t in (x, w.reshape(1, H), b))
    pool, local = ops.pool_local(xr, probs[:, None], pnn[:, None], batch, wr, br, B)
    pool_ref, local_ref = _pool_ref(x.double(), probs, pnn, batch, w, b, B)
    assert pool.shape == (B, H) and torch.equal(pool.double(), pool_ref)
    assert torch.equal(local.reshape(-1).double(), local_ref)
    (pool * dpool).sum().add_((local.reshape(-1) * dlocal).sum()).backward()
    dx_ref, dw_ref, db_ref = _pool_bwd_ref(x.double(), probs, pnn, batch, w, dpool, dlocal, B, torch.zeros(H, device="cuda"),
                                           torch.zeros(1, device="cuda"))
    assert xr.grad.shape == (len(batch), H) and torch.equal(xr.grad.double(), dx_ref)
    assert wr.grad.shape == (1, H) and torch.equal(wr.grad.reshape(-1).double(), dw_ref)
    assert torch.equal(br.grad.double(), db_ref.reshape(1))


def test_global_add_pool_follows_pyg():
    """batch=None sums every row into one graph ([1, H]); a width above 256 is refused (pert_model_width)."""
    from pert_gnn_kdd23_b200 import _lib, nn

    g = torch.Generator().manual_seed(0)
    for H in (3, 64):
        x = torch.randint(-4, 5, (1001, H), generator=g).float().cuda()
        got = nn.global_add_pool(x, None)
        assert got.shape == (1, H) and torch.equal(got.double(), x.double().sum(0, keepdim=True))
        got = nn.global_add_pool(x, None, size=5)          # PyG ignores size without a batch vector
        assert got.shape == (1, H)
        batch, B = _graph_layout([500, 1, 500])
        got = nn.global_add_pool(x, batch.cuda())
        want = torch.zeros(B, H, dtype=torch.float64).index_add_(0, batch, x.double().cpu())
        assert torch.equal(got.double().cpu(), want)
    with pytest.raises(_lib.PertGnnError):
        nn.global_add_pool(torch.ones(8, 260, device="cuda"), torch.zeros(8, dtype=torch.int64, device="cuda"), 1)


# ==================================================================================================== embeddings
def _ids_matrix(ids_col, stride, col, g, n_rows):
    """[N, stride] int64 matrix whose column `col` holds the ids (the other columns other tables' ids)."""
    m = torch.randint(0, n_rows, (ids_col.numel(), stride), generator=g)
    m[:, col] = ids_col
    return m.cuda()


def _emb_fwd(table, idm, col, N, H, ld_out, out=None, accumulate=0):
    L = _L()
    if out is None:
        out = torch.full((N + 2, ld_out), SENT, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc = L.pert_embedding_fwd(table.data_ptr(), table.size(0), idm.data_ptr() + 8 * col, idm.size(1), out.data_ptr(),
                              ld_out, N, H, accumulate, status.data_ptr(), _st())
    torch.cuda.synchronize()
    return rc, out, int(status)


def _emb_bwd(dybuf, idm, col, dtable, N, H):
    rc = _L().pert_embedding_bwd(dybuf.data_ptr(), dybuf.stride(0), idm.data_ptr() + 8 * col, idm.size(1),
                                 dtable.data_ptr(), dtable.size(0), N, H, _st())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("H", [4, 12, 64, 100, 256])
@pytest.mark.parametrize("stride", [1, 2, 3, 4])
def test_embedding_fwd_gather_and_table_sum(H, stride):
    """The gather is bit-exact; accumulate = 1 over up to four tables equals the fp32 sum in table order; ids from one
    column of a [N, stride] matrix (cat_X), ld_out > H."""
    g = torch.Generator().manual_seed(H * 5 + stride)
    N, ld = 1037, H + 8
    tables = [torch.randn(r, H, generator=g).cuda() for r in (17, 3, 40, 9)][:stride]
    idm = torch.stack([torch.randint(0, t.size(0), (N,), generator=g) for t in tables], 1).cuda()
    out = None
    want = None
    for i, t in enumerate(tables):
        rc, out, status = _emb_fwd(t, idm, i, N, H, ld, out=out, accumulate=int(i > 0))
        assert rc == 0 and status == 0
        rows = t[idm[:, i]]
        want = rows if want is None else rows + want
        assert torch.equal(out[:N, :H], want), f"table {i} (H={H} stride={stride})"
        _untouched(out, N, H, f"embedding out, table {i}")


def test_embedding_fwd_out_of_range_ids_report():
    """A negative id and an id >= n_rows set the status word; every other row is still gathered exactly."""
    g = torch.Generator().manual_seed(0)
    H, N = 32, 500
    table = torch.randn(10, H, generator=g).cuda()
    for bad in (-1, 10, 1 << 40):
        ids = torch.randint(0, 10, (N,), generator=g)
        ids[123] = bad
        idm = ids[:, None].cuda()
        rc, out, status = _emb_fwd(table, idm, 0, N, H, H)
        assert rc == 0 and status == RANGE, bad
        keep = torch.arange(N, device="cuda") != 123
        assert torch.equal(out[:N][keep], table[idm[keep, 0]])
        _untouched(out, N, H, "embedding out")


def _run_ids(pattern, N, n_rows, g):
    if pattern == "runs":           # run lengths 1..20: shorter than, equal to and longer than EB_RUN
        lens = torch.randint(1, 21, (N,), generator=g)
        ids = torch.repeat_interleave(torch.randint(0, n_rows, (N,), generator=g), lens)[:N]
    elif pattern == "runs_of_8":    # runs of exactly EB_RUN, offset by 3 so each crosses a chunk boundary
        ids = (torch.arange(N) + 3) // EB_RUN % n_rows
    elif pattern == "alternating":
        ids = torch.arange(N) % 2
    elif pattern == "hot":
        ids = torch.full((N,), 3)
    else:                           # random
        ids = torch.randint(0, n_rows, (N,), generator=g)
    return ids.to(torch.int64)


@pytest.mark.parametrize("pattern", ["runs", "runs_of_8", "alternating", "hot", "random"])
@pytest.mark.parametrize("H", [4, 64, 100])
@pytest.mark.parametrize("N", [7, 8, 9, 1001, 100_003])
def test_embedding_bwd_runs(pattern, H, N):
    """Scatter-add of integer gradients into a non-zero table, bit-exact: runs of equal ids shorter than, equal to and
    longer than EB_RUN across the 8-row chunks, alternating ids, one hot row taking every node; ids read from column 1
    of a [N, 3] matrix, ld_dy > H."""
    g = torch.Generator().manual_seed(N + H)
    n_rows = 50
    ids = _run_ids(pattern, N, n_rows, g)
    idm = _ids_matrix(ids, 3, 1, g, n_rows)
    dy = torch.randint(-4, 5, (N, H), generator=g).float().cuda()
    dt0 = torch.randint(-3, 4, (n_rows, H), generator=g).float().cuda()
    dt = dt0.clone()
    assert _emb_bwd(_strided(dy, H + 4), idm, 1, dt, N, H) == 0
    want = dt0.double().index_add_(0, idm[:, 1], dy.double())
    assert torch.equal(dt.double(), want), f"{pattern} N={N} H={H}"


def test_embedding_bwd_drops_out_of_range_ids():
    g = torch.Generator().manual_seed(1)
    H, N, n_rows = 16, 333, 9
    ids = torch.randint(0, n_rows, (N,), generator=g)
    ids[[0, 1, 40, 41, 42, 100, 332]] = torch.tensor([-1, -1, n_rows, n_rows, 5, -3, n_rows + 7])
    idm = ids[:, None].cuda()
    dy = torch.randint(-4, 5, (N, H), generator=g).float().cuda()
    dt = torch.zeros(n_rows + 2, H, device="cuda")        # two spare rows: an id >= n_rows must not land there
    dt[n_rows:] = SENT
    rc = _L().pert_embedding_bwd(dy.data_ptr(), H, idm.data_ptr(), 1, dt.data_ptr(), n_rows, N, H, _st())
    torch.cuda.synchronize()
    assert rc == 0
    ok = (ids >= 0) & (ids < n_rows)
    want = torch.zeros(n_rows, H, dtype=torch.float64).index_add_(0, ids[ok], dy.double().cpu()[ok])
    assert torch.equal(dt[:n_rows].double().cpu(), want) and bool((dt[n_rows:] == SENT).all())


@pytest.mark.parametrize("H", [1, 5, 13, 64])
def test_embedding_ops_any_width(H):
    """ops.embedding at H % 4 != 0 (zero-padded to whole float4s): the gather and the scatter-add of integer
    gradients bit-exact, shapes of H."""
    from pert_gnn_kdd23_b200 import ops

    g = torch.Generator().manual_seed(H)
    N, n_rows = 2049, 30
    table = torch.randn(n_rows, H, generator=g).cuda().requires_grad_()
    ids = _run_ids("runs", N, n_rows, g)
    idm = _ids_matrix(ids, 4, 2, g, n_rows)
    out = ops.embedding(table, idm, col=2)
    assert out.shape == (N, H) and torch.equal(out, table.detach()[idm[:, 2]])
    dy = torch.randint(-4, 5, (N, H), generator=g).float().cuda()
    out.backward(dy)
    want = torch.zeros(n_rows, H, dtype=torch.float64, device="cuda").index_add_(0, idm[:, 2], dy.double())
    assert table.grad.shape == (n_rows, H) and torch.equal(table.grad.double(), want)


@pytest.mark.parametrize("H,F", [(64, 16), (5, 3), (32, 0), (12, 7)])
def test_embed_concat_layout(H, F):
    """X0 = [sum_i table_i[cat_X[:, i]] | x | 0-pad] with ld = round_up(H + F, 8): the embedding block is the fp32 sum in
    table order, x is copied exactly, the pad columns are exactly 0; gradients bit-exact on integer data."""
    from pert_gnn_kdd23_b200 import ops

    g = torch.Generator().manual_seed(H + F)
    N = 1500
    rows = (11, 4, 23)
    tables = [torch.randn(r, H, generator=g).cuda().requires_grad_() for r in rows]
    cat_X = torch.stack([torch.randint(0, r, (N,), generator=g) for r in rows], 1).cuda()
    x = torch.randn(N, F, generator=g).cuda().requires_grad_()
    out = ops.embed_concat(x, cat_X, tables)
    ld = (H + F + 7) // 8 * 8
    assert out.shape == (N, ld)
    want = None
    for i, t in enumerate(tables):
        r = t.detach()[cat_X[:, i]]
        want = r if want is None else r + want
    assert torch.equal(out[:, :H], want)
    assert torch.equal(out[:, H:H + F], x.detach())
    assert bool((out[:, H + F:] == 0).all()) and not bool(torch.signbit(out[:, H + F:]).any())
    dout = torch.randint(-4, 5, (N, ld), generator=g).float().cuda()
    out.backward(dout)
    for i, t in enumerate(tables):
        w = torch.zeros(rows[i], H, dtype=torch.float64, device="cuda").index_add_(0, cat_X[:, i], dout[:, :H].double())
        assert torch.equal(t.grad.double(), w), f"table {i}"
    assert torch.equal(x.grad, dout[:, H:H + F])


def test_copy_cols():
    """out[:, col0:col0+F] = x, out[:, col0+F:ld] = 0, columns below col0 untouched."""
    g = torch.Generator().manual_seed(0)
    N, F, col0, ld = 777, 9, 12, 24
    x = torch.randn(N, F, generator=g).cuda()
    out = torch.full((N + 2, ld), SENT, device="cuda")
    rc = _L().pert_copy_cols(x.data_ptr(), F, out.data_ptr(), ld, col0, N, _st())
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.equal(out[:N, col0:col0 + F], x) and bool((out[:N, col0 + F:] == 0).all())
    assert bool((out[:N, :col0] == SENT).all()) and bool((out[N:] == SENT).all())
