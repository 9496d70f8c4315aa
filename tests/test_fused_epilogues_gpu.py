"""The LayerNorm-fused GEMM epilogues, the head-major value store and the LayerNorm variants, kernel by kernel against float64
(lwdetr_gemm_ex, lwdetr_layernorm_ex).

Reference: float64 torch on the same 16-bit operands the kernels read.  Every bound is built per element from the data:
  output rounding      half an ulp of the 16-bit result;
  accumulation         wgmma adds each k16 step's 16 exact products of 16-bit operands to the fp32 accumulator; a step loses at
                       most 2 fp32 ulps (alignment to the largest term, then rounding) of a value no larger than S = sum_k |a_k w_k|,
                       so K/16 steps stay within ACC * S with ACC = K/16 * 2^-22;
  fp32 epilogue        a few fp32 roundings (2^-21 relative) of the epilogue's intermediate values, written out term by term below.
The LayerNorm consumer multiplies the accumulation term by rstd: on a row whose mean is large against its spread, acc and
mean * colsum cancel and the fold's error is rstd * ACC * S, which the test reports in fp16 half-ulps of the output."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
RAN = set()          # (epilogue, bn, dtype) instances and LayerNorm rows-per-warp instances that ran
FOLD_HALF_ULPS = {}  # (mean/spread ratio, GELU) -> worst fp16 LN-fold error in half-ulps of max(|output|, 1)
# Cap on that error per mean/spread ratio, fp16 (DESIGN.md 3.1).  The analytical bound of _check_consumer holds for every row, but
# on rows whose mean is large against their spread it is loose (rstd * K/16 * 2^-22 * sum|x W'| reaches ~2000 half-ulps at C = 768
# and ratio 4000), so these rows are also held to the error the H100 measured with this file's data: worst over C = 192 / 384 /
# 768 and every part count, 1.0 / 2.4 / 13.5 / 44.2 half-ulps at ratio 1 / 1e2 / 1e3 / 4e3.  The caps are twice that, rounded
# up: the error comes from the accumulator's alignment and truncation of the exact products, which varies with the data, and
# twice the worst of ~2800 rows per ratio leaves room for other rows without letting through a term carried with 1e-4 relative
# error (about 800 half-ulps on a mean-1000 row).  The GELU epilogue scales the pre-activation error by at most |gelu'| <= 1.13
# and adds its polynomial's 7.4e-5 (0.15 half-ulps at 1): 1.13 * cap + 0.5.
FOLD_CAP_HALF_ULPS = {1.0: 2.0, 1e2: 5.0, 1e3: 27.0, 4e3: 89.0}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    cm = request.config.pluginmanager.get_plugin("capturemanager")
    if tr is None or cm is None:
        return
    with cm.global_and_fixture_disabled():
        _write_report(tr)


def _write_report(tr):
    tr.write_line("")
    tr.write_line("fused epilogue instances run: " + ", ".join("%s/BN%d/%s" % (e, b, d) for e, b, d in
                                                            sorted(x for x in RAN if x[0].startswith("EP"))))
    tr.write_line("layernorm instances run: " + ", ".join("RPW%d/C%d/%s" % (r, c, d) for _, r, c, d in
                                                       sorted(x for x in RAN if x[0] == "LN")))
    for (ratio, gelu) in sorted(FOLD_HALF_ULPS):
        tr.write_line("LN-fold worst error, fp16, %s, mean/spread ~%g: %.2f half-ulps of max(|output|, 1) (cap %.1f)" % (
            "EP_LN_GELU" if gelu else "EP_LN", ratio, FOLD_HALF_ULPS[ratio, gelu], _fold_cap(ratio, gelu)))


def _fold_cap(ratio, gelu):
    cap = FOLD_CAP_HALF_ULPS[ratio]
    return 1.13 * cap + 0.5 if gelu else cap


def _dn(dt):
    return str(dt).split(".")[-1]


def _stats_buf(M):
    """NaN-filled room for the partials of M rows at any part count (at most 48); _stats_rows views it as the kernel writes it."""
    return torch.full(((M + 3) * 48 * 2,), float("nan"), device="cuda", dtype=torch.float32)


def _stats_rows(buf, M, parts):
    """[M + 3, parts, 2] view of a _stats_buf (the producer writes row m's partials at m * parts), and the untouched rest."""
    n = (M + 3) * parts * 2
    return buf[:n].view(M + 3, parts, 2), buf[n:]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _pick_bn(N, m_tiles):
    """The tile width gemm_build chooses (gemm_tc.cu pick_bn), restated to choose shapes that land on each width."""
    waste = lambda b: -(-N // b) * b - N
    if N <= 64:
        bn = 64
    elif N <= 128:
        bn = 128
    else:
        bn = min((256, 192, 128), key=lambda c: (waste(c), (256, 192, 128).index(c)))
    while bn > 64 and m_tiles * -(-N // bn) < _sms():
        nb = 128 if bn == 256 else 64
        if waste(nb) > waste(bn) + 32:
            break
        bn = nb
    return bn


def _half_ulp(v, dt):
    """Half an ulp of the 16-bit format at |v| (float64 tensor), one binade up so that a result rounded across a power of two
    is covered."""
    mant, emin = (10, -14) if dt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(v.abs() * (1 + 2.0 ** -8) + 2.0 ** (emin - 1))).clamp(min=emin)
    return torch.exp2(e - mant - 1)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# --------------------------------------------------------------------------------------------------- row kinds
RATIOS = {torch.float16: (1.0, 1e2, 1e3, 4e3), torch.bfloat16: (1.0, 10.0, 30.0, 60.0)}   # bf16 cannot hold 0.25 spread at 1000


def _kind_rows(M, C, dt, g, spread=0.25):
    """Raw LayerNorm input rows: normal rows, rows of mean ratio*spread and spread `spread` for each ratio in RATIOS[dt] (the
    last fp16 ratio is mean 1000), constant rows (variance 0: eps governs) and rows with one channel at +-500 (a "massive
    activation").  Returns (x 16-bit [M, C], ratio per row (0 = not a ratio row), kind per row)."""
    x = torch.randn(M, C, device="cuda", generator=g) * 0.8 + 0.3
    r = torch.arange(M, device="cuda")
    ratio = torch.zeros(M, device="cuda", dtype=torch.float64)
    kind = torch.zeros(M, device="cuda", dtype=torch.long)
    for j, q in enumerate(RATIOS[dt]):
        sel = r % 16 == 3 + 2 * j
        x[sel] = q * spread + spread * torch.randn(int(sel.sum()), C, device="cuda", generator=g)
        ratio[sel] = q
        kind[sel] = 1 + j
    sel = r % 16 == 11
    x[sel] = 3.0
    kind[sel] = 5
    sel = (r % 16 == 13).nonzero().flatten()
    x[sel, sel % C] = torch.where(sel % 2 == 0, 500.0, -500.0).to(x.dtype)
    kind[sel] = 6
    return x.to(dt), ratio, kind


def _partials64(x64, parts):
    """(sum, M2) over `parts` equal column slices per row, float64."""
    xs = x64.view(x64.shape[0], parts, -1)
    return torch.stack([xs.sum(dim=2), ((xs - xs.mean(dim=2, keepdim=True)) ** 2).sum(dim=2)], dim=2)


def _combine64(st, C):
    """Chan-style combination of equal-width partials [M, parts, 2] in float64 -> (mean, biased variance)."""
    st = st.double()
    n_p = C / st.shape[1]
    mean = st[:, :, 0].sum(dim=1) / C
    var = (st[:, :, 1].sum(dim=1) + n_p * ((st[:, :, 0] / n_p - mean[:, None]) ** 2).sum(dim=1)) / C
    return mean, var


def _gelu64(v):
    return 0.5 * v * (1.0 + torch.erf(v / 2 ** 0.5))


# --------------------------------------------------------------------------------------------------- LayerNorm consumer
def _fold(C, N, dt, g, wscale=1.0):
    """W' (LayerNorm weight folded in, rounded to dt), colsum = sum of the ROUNDED W' (engine.cpp fold_ln), bias' fp32."""
    W = torch.randn(N, C, device="cuda", generator=g) / C ** 0.5 * wscale
    lnw = torch.rand(C, device="cuda", generator=g) + 0.5
    lnb = torch.randn(C, device="cuda", generator=g) * 0.2
    bias = torch.randn(N, device="cuda", generator=g) * 0.3
    Wf = (W * lnw).to(dt)
    cs = Wf.double().sum(dim=1).float()
    bf = (bias.double() + W.double() @ lnb.double()).float()
    return Wf, cs, bf


def _check_consumer(x, stats_in, Wf, cs, bf, out, gelu, dt, ratio=None, eps=1e-6, what=""):
    """out (device) against float64 LayerNorm -> linear on the rounded rows x, with mean / var taken from x itself."""
    x64 = x.double()
    C = x64.shape[1]
    mean = x64.mean(dim=1, keepdim=True)
    var = x64.var(dim=1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    W64 = Wf.double()
    acc = x64 @ W64.t()
    pre = rstd * (acc - mean * cs.double()) + bf.double()
    ref = _gelu64(pre) if gelu else pre
    S = x64.abs() @ W64.abs().t()
    ACC = C / 16 * 2.0 ** -22
    e_pre = rstd * (ACC * S + mean.abs() * cs.double().abs() * 2.0 ** -21 + acc.abs() * 2.0 ** -22) \
        + (pre - bf.double()).abs() * 2.0 ** -20 + bf.double().abs() * 2.0 ** -23
    if gelu:
        e_pre = 1.13 * e_pre + 8e-5 * torch.clamp(pre.abs(), min=1.0)   # |gelu'| <= 1.13; polynomial (epilogue.cuh gelu_erf2)
    hu = _half_ulp(ref, dt)
    err = (out.double() - ref).abs()
    bad = ~(err <= e_pre + hu)
    assert not bad.any(), "%s: %d elements out of bound, worst row %d err %.4g bound %.4g" % (
        what, int(bad.sum()), int(bad.nonzero()[0, 0]), float(err[bad].max()), float((e_pre + hu)[bad].max()))
    if dt == torch.float16 and ratio is not None:
        for q in RATIOS[dt]:
            sel = ratio == q
            if sel.any():
                # in half-ulps of an O(1) output: elements near zero would inflate a per-element ratio
                hu1 = _half_ulp(torch.clamp(ref[sel].abs(), min=1.0), dt)
                worst = float((err[sel] / hu1).max())
                FOLD_HALF_ULPS[q, gelu] = max(FOLD_HALF_ULPS.get((q, gelu), 0.0), worst)
                assert worst <= _fold_cap(q, gelu), "%s: LN-fold error %.1f half-ulps on rows of mean/spread %g, cap %.1f" % (
                    what, worst, q, _fold_cap(q, gelu))
    return err, hu


CONSUMER_CASES = [(C, parts) for C, ps in ((192, (2, 6)), (384, (4, 12)), (768, (6, 12, 24))) for parts in ps]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C,parts", CONSUMER_CASES)
@pytest.mark.parametrize("mult", [3, 4])     # qkv: N = 3C, EP_LN; fc1: N = 4C, EP_LN_GELU
def test_layernorm_consumer_matches_float64(dt, C, parts, mult):
    from b200 import capi
    g = _gen(1000 * C + 10 * parts + mult)
    M = 3200 + 77                                     # ragged: not a multiple of 128
    ntap = 3
    xw = torch.zeros(M, ntap * C, device="cuda", dtype=dt)
    x, ratio, _ = _kind_rows(M, C, dt, g)
    xw[:, C:2 * C] = x                                 # a column slice of a tap buffer: lda = ntap * C
    xs = xw[:, C:2 * C]
    stats_in = _partials64(x.double(), parts).float().contiguous()
    N = mult * C
    Wf, cs, bf = _fold(C, N, dt, g)
    out = torch.full((M + 5, N), float("nan"), device="cuda", dtype=dt)
    gelu = mult == 4
    bn, ep, _ = capi.gemm_ex(xs, Wf, out, bias=bf, act=capi.ACT_GELU if gelu else capi.ACT_NONE, M=M, stats_in=stats_in, colsum=cs,
                             ln_C=C, ln_eps=1e-6)
    torch.cuda.synchronize()
    assert ep == ("EP_LN_GELU" if gelu else "EP_LN") and bn == _pick_bn(N, -(-M // 128))
    RAN.add((ep, bn, _dn(dt)))
    assert torch.isnan(out[M:]).all(), "wrote past row M"
    _check_consumer(x, stats_in, Wf, cs, bf, out[:M], gelu, dt, ratio, what="C=%d parts=%d N=%d" % (C, parts, N))


def test_layernorm_consumer_all_tile_widths():
    """EP_LN and EP_LN_GELU at every width pick_bn can choose for them: the engine's N = 3C / 4C at large and small M."""
    from b200 import capi
    seen = set()
    for dt in DTYPES:
        for C, N in ((192, 576), (192, 768), (384, 1152), (384, 1536), (768, 2304), (768, 3072), (256, 512)):
            for M in (128 * _sms() + 37, 1000):
                g = _gen(C + N + M)
                x, ratio, _ = _kind_rows(M, C, dt, g)
                Wf, cs, bf = _fold(C, N, dt, g)
                stats_in = _partials64(x.double(), 2).float().contiguous()
                for gelu in (False, True):
                    out = torch.empty(M, N, device="cuda", dtype=dt)
                    bn, ep, _ = capi.gemm_ex(x, Wf, out, bias=bf, act=capi.ACT_GELU if gelu else capi.ACT_NONE, stats_in=stats_in,
                                             colsum=cs, ln_C=C, ln_eps=1e-6)
                    torch.cuda.synchronize()
                    RAN.add((ep, bn, _dn(dt)))
                    seen.add((ep, bn))
                    _check_consumer(x, stats_in, Wf, cs, bf, out, gelu, dt, ratio, what="C=%d N=%d M=%d" % (C, N, M))
    for ep in ("EP_LN", "EP_LN_GELU"):
        assert {b for e, b in seen if e == ep} == {64, 128, 192, 256}, seen


# --------------------------------------------------------------------------------------------------- statistics producer
def _producer_inputs(M, C, K, dt, g, resid_rows, affine):
    """A [M, K], W [C, K], a residual table [resid_rows, C] with the row kinds of _kind_rows in its rows (A rows of constant-kind
    rows are zero, of mean-1000 rows small, so that the output row keeps its kind), bias / gamma or None."""
    A = torch.randn(M, K, device="cuda", generator=g)
    W = (torch.randn(C, K, device="cuda", generator=g) / K ** 0.5).to(dt)
    resid, _, kind = _kind_rows(resid_rows, C, dt, g)
    rk = kind[torch.arange(M, device="cuda") % resid_rows]
    A[rk == 5] = 0.0
    A[(rk >= 1) & (rk <= 4)] *= 0.01
    bias = torch.randn(C, device="cuda", generator=g) * 0.2 if affine else None
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5 if affine else None
    return A.to(dt), W, resid, bias, gamma, rk


def _check_producer(A, W, resid, resid_mod, bias, gamma, out, stats, parts, dt, M, rk, what):
    C = W.shape[0]
    K = A.shape[1]
    rows = torch.arange(M, device="cuda") % (resid_mod if resid_mod else M)
    r64 = resid.double()[rows]
    acc = A.double() @ W.double().t()
    g64 = gamma.double() if gamma is not None else torch.ones(C, device="cuda", dtype=torch.float64)
    b64 = bias.double() if bias is not None else torch.zeros(C, device="cuda", dtype=torch.float64)
    ref = r64 + g64 * (acc + b64)
    S = A.double().abs() @ W.double().abs().t()
    bound = _half_ulp(ref, dt) + g64.abs() * (K / 16 * 2.0 ** -22 * S + (acc + b64).abs() * 2.0 ** -22) + ref.abs() * 2.0 ** -23
    o64 = out.double()
    err = (o64 - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), "%s: %d elements out of bound, err %.4g" % (what, int(bad.sum()), float(err[bad].max()))
    if gamma is None and bias is None:
        const = rk == 5
        assert (o64[const] == o64[const][:, :1]).all(), "constant rows are not constant"
    # every partial: (sum, M2) of the ROUNDED output over its own C / parts columns.  Partial 2 * t + h belongs to n-tile t and
    # column half h: the 32-column groups 2 * pass + h of each 64-column epilogue pass, shifted by its first value
    st = stats[:M].double()
    assert torch.isfinite(st).all(), "%s: a partial slot was not written (or two collided)" % what
    bn = 2 * C // parts
    cols = torch.tensor([t * bn + 64 * pc + 32 * h + j for t in range(parts // 2) for h in range(2) for pc in range(bn // 64)
                         for j in range(32)], device="cuda")
    xs = o64[:, cols].view(M, parts, C // parts)
    x0 = xs[:, :, :1]
    s_ref = xs.sum(dim=2)
    m2_ref = ((xs - xs.mean(dim=2, keepdim=True)) ** 2).sum(dim=2)
    tol_s = 2.0 ** -16 * (xs - x0).abs().sum(dim=2) + 2.0 ** -22 * s_ref.abs() + 1e-30
    tol_m2 = 2.0 ** -16 * ((xs - x0) ** 2).sum(dim=2) + 1e-30
    assert ((st[:, :, 0] - s_ref).abs() <= tol_s).all(), "%s: partial sums" % what
    assert ((st[:, :, 1] - m2_ref).abs() <= tol_m2).all(), "%s: partial M2" % what
    mean, var = _combine64(st, C)
    assert torch.allclose(mean, o64.mean(dim=1), rtol=1e-5, atol=1e-5), what
    assert torch.allclose(var, o64.var(dim=1, unbiased=False), rtol=1e-4, atol=1e-5), what
    assert torch.isnan(stats[M:]).all(), "%s: statistics written past row M" % what


PRODUCER_CASES = [(C, size) for C in (192, 384, 768) for size in ("large", "small")] + [(768, "medium")]
PRODUCER_M = {"large": lambda: 128 * _sms() + 37, "medium": lambda: 128 * 30 + 11, "small": lambda: 128 * 6 + 19}


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C,size", PRODUCER_CASES)
@pytest.mark.parametrize("form", ["proj", "patch_embed", "fc2"])
def test_statistics_producer_matches_float64(dt, C, size, form):
    """proj (K = C, residual + gamma, out into a column slice of a tap buffer), patch_embed (K = 768, a position table as the
    residual with resid_mod, and gamma), fc2 (K = 4C, no affine, so the constant rows stay constant)."""
    from b200 import capi
    g = _gen(C * 7 + len(form) + len(size))
    M = PRODUCER_M[size]()
    K = {"proj": C, "patch_embed": 768, "fc2": 4 * C}[form]
    resid_rows = 1600 if form == "patch_embed" else M
    A, W, resid, bias, gamma, rk = _producer_inputs(M, C, K, dt, g, resid_rows, affine=form != "fc2")
    ntap = 3
    outw = torch.full((M + 3, ntap * C), float("nan"), device="cuda", dtype=dt)
    out = outw[:, C:2 * C]                                                   # ld_out = ntap * C
    buf = _stats_buf(M)
    bn, ep, parts = capi.gemm_ex(A, W, out, bias=bias, gamma=gamma, resid=resid, resid_mod=resid_rows if form == "patch_embed" else 0,
                                 M=M, stats_out=buf)
    stats, rest = _stats_rows(buf, M, parts)
    torch.cuda.synchronize()
    assert ep == "EP_RESID" and bn == _pick_bn(C, -(-M // 128)) and parts == 2 * (C // bn), (bn, ep, parts)
    RAN.add(("EP_RESID+stats", bn, _dn(dt)))
    assert torch.isnan(outw[:, :C]).all() and torch.isnan(outw[:, 2 * C:]).all(), "wrote outside its column slice"
    assert torch.isnan(outw[M:]).all(), "wrote past row M"
    assert torch.isnan(rest).all(), "statistics written past row M"
    _check_producer(A, W, resid, resid_rows if form == "patch_embed" else 0, bias, gamma, out[:M], stats, parts, dt, M, rk,
                    "%s C=%d M=%d" % (form, C, M))


# --------------------------------------------------------------------------------------------------- specialised == generic
SPEC_SHAPES = {256: 512, 192: 576, 128: 640, 64: 192}   # N per tile width (the 64 case narrows at small M)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("ep", ["EP_BIAS", "EP_BIAS_ACT", "EP_LN", "EP_LN_GELU", "EP_RESID", "EP_RESID+stats"])
def test_specialised_epilogue_equals_generic(dt, bn, ep):
    """An all-zero row_zero vector forces EP_GENERIC without changing the math: outputs and partials must be bit-identical."""
    from b200 import capi
    g = _gen(bn * 31 + len(ep))
    N = SPEC_SHAPES[bn]
    M = 128 * 8 + 45 if bn == 64 else 128 * _sms() + 45
    C = 256
    x, _, _ = _kind_rows(M, C, dt, g)
    kw = {}
    if ep in ("EP_LN", "EP_LN_GELU"):
        Wf, cs, bf = _fold(C, N, dt, g)
        kw = dict(bias=bf, stats_in=_partials64(x.double(), 4).float().contiguous(), colsum=cs, ln_C=C, ln_eps=1e-6,
                  act=capi.ACT_GELU if ep == "EP_LN_GELU" else capi.ACT_NONE)
    else:
        Wf = (torch.randn(N, C, device="cuda", generator=g) / C ** 0.5).to(dt)
        kw = dict(bias=torch.randn(N, device="cuda", generator=g) * 0.3)
        if ep == "EP_BIAS_ACT":
            kw["act"] = capi.ACT_GELU
        if ep.startswith("EP_RESID"):
            kw["gamma"] = torch.rand(N, device="cuda", generator=g) + 0.5
            kw["resid"] = (torch.randn(M, N, device="cuda", generator=g) * 2).to(dt)
    outs, stats = [], []
    for rz in (None, torch.zeros(M, device="cuda", dtype=torch.uint8)):
        out = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
        st = _stats_buf(M) if ep == "EP_RESID+stats" else None
        b, e, _ = capi.gemm_ex(x, Wf, out, row_zero=rz, stats_out=st, **kw)
        assert b == bn, (b, bn)
        assert e == (ep.split("+")[0] if rz is None else "EP_GENERIC"), e
        outs.append(out)
        stats.append(st)
    torch.cuda.synchronize()
    RAN.add((ep, bn, _dn(dt)))
    assert not torch.isnan(outs[0]).any()
    assert torch.equal(outs[0], outs[1]), "specialised %s differs from the generic epilogue in %d elements" % (
        ep, int((outs[0] != outs[1]).sum()))
    if stats[0] is not None:
        assert torch.equal(torch.nan_to_num(stats[0], nan=7.0), torch.nan_to_num(stats[1], nan=7.0)), "partials differ"


# --------------------------------------------------------------------------------------------------- producer -> consumer chains
def _stats_view(buf, M, parts):
    return _stats_rows(buf, M, parts)[0][:M]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C", [192, 384, 768])
@pytest.mark.parametrize("M", [3200, 128 * 7 + 5])
def test_producer_to_consumer_chain(dt, C, M):
    """patch_embed-style producer -> qkv consumer, then proj producer -> fc1 consumer, with the partials the device wrote."""
    from b200 import capi
    g = _gen(C + M)
    A, W, pos, bias, _, _ = _producer_inputs(M, C, 768, dt, g, 1600, affine=True)
    x = torch.empty(M, C, device="cuda", dtype=dt)
    st = _stats_buf(M)
    _, _, parts = capi.gemm_ex(A, W, x, bias=bias, resid=pos, resid_mod=1600, stats_out=st)
    Wq, csq, bq = _fold(C, 3 * C, dt, g)
    qkv = torch.empty(M, 3 * C, device="cuda", dtype=dt)
    sv = _stats_view(st, M, parts)
    capi.gemm_ex(x, Wq, qkv, bias=bq, stats_in=sv, colsum=csq, ln_C=C, ln_eps=1e-6)
    torch.cuda.synchronize()
    _check_consumer(x, sv, Wq, csq, bq, qkv, False, dt, what="patch_embed -> qkv C=%d parts=%d" % (C, parts))
    # proj producer (residual x, gamma) -> fc1 consumer
    att = (torch.randn(M, C, device="cuda", generator=g)).to(dt)
    Wp = (torch.randn(C, C, device="cuda", generator=g) / C ** 0.5).to(dt)
    gam = torch.rand(C, device="cuda", generator=g) * 0.5
    xm = torch.empty(M, C, device="cuda", dtype=dt)
    st2 = _stats_buf(M)
    _, _, parts2 = capi.gemm_ex(att, Wp, xm, bias=bias, gamma=gam, resid=x, stats_out=st2)
    W1, cs1, b1 = _fold(C, 4 * C, dt, g)
    h = torch.empty(M, 4 * C, device="cuda", dtype=dt)
    sv2 = _stats_view(st2, M, parts2)
    capi.gemm_ex(xm, W1, h, bias=b1, act=capi.ACT_GELU, stats_in=sv2, colsum=cs1, ln_C=C, ln_eps=1e-6)
    torch.cuda.synchronize()
    _check_consumer(xm, sv2, W1, cs1, b1, h, True, dt, what="proj -> fc1 C=%d parts=%d" % (C, parts2))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("M", [3200, 17000])       # fc2 at BN 64 (6 partials) and BN 192 (2 partials) on 132 SMs
def test_fc2_to_mlp_to_qkv_chain(dt, M):
    """C = 192: fc2 producer (BN 192 at large M, 64 at small) -> fused-MLP consumer (its own partials out) -> qkv consumer."""
    from b200 import capi
    C = 192
    g = _gen(M)
    hid = (torch.randn(M, 4 * C, device="cuda", generator=g) * 0.5).to(dt)
    W2 = (torch.randn(C, 4 * C, device="cuda", generator=g) / (4 * C) ** 0.5).to(dt)
    xr, _, _ = _kind_rows(M, C, dt, g)
    b2 = torch.randn(C, device="cuda", generator=g) * 0.1
    g2 = torch.rand(C, device="cuda", generator=g) + 0.5
    x = torch.empty(M, C, device="cuda", dtype=dt)
    st = _stats_buf(M)
    bn, _, parts = capi.gemm_ex(hid, W2, x, bias=b2, gamma=g2, resid=xr, stats_out=st)
    assert bn == _pick_bn(C, -(-M // 128)) and parts in (2, 6)
    sv = _stats_view(st, M, parts)
    W1, cs1, b1 = _fold(C, 4 * C, dt, g)
    W2b = (torch.randn(C, 4 * C, device="cuda", generator=g) / (4 * C) ** 0.5).to(dt)
    y = torch.empty(M, C, device="cuda", dtype=dt)
    st_y = torch.full((M, parts, 2), float("nan"), device="cuda")
    capi.vit_mlp(x, sv, W1, cs1, b1, W2b, b2=b2, gamma=g2, out=y, stats_out=st_y)
    torch.cuda.synchronize()
    # float64 LN -> fc1 -> GELU -> round -> fc2 -> gamma, residual, on the device's x
    x64 = x.double()
    mean, var = x64.mean(dim=1, keepdim=True), x64.var(dim=1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    pre = rstd * (x64 @ W1.double().t() - mean * cs1.double()) + b1.double()
    h64 = _gelu64(pre).to(dt).double()
    branch = h64 @ W2b.double().t() + b2.double()
    ref = x64 + g2.double() * branch
    # the hidden value is rounded in both: a one-ulp disagreement of h (fold error) moves the branch by |W2| * ulp(h)
    e_h = 1.13 * (rstd * (C / 16 * 2.0 ** -22 * (x64.abs() @ W1.double().abs().t()) + mean.abs() * cs1.double().abs() * 2.0 ** -21)
                  + (pre - b1.double()).abs() * 2.0 ** -20) + 8e-5 * torch.clamp(pre.abs(), min=1.0) + 2 * _half_ulp(h64, dt)
    bound = _half_ulp(ref, dt) + g2.double() * (e_h @ W2b.double().abs().t() + 48 * 2.0 ** -22 * (h64.abs() @ W2b.double().abs().t())
                                                + branch.abs() * 2.0 ** -22)
    err = (y.double() - ref).abs()
    assert (err <= bound).all(), "fc2 -> mlp: worst err %.4g" % float(err.max())
    mean_y, var_y = _combine64(st_y, C)
    assert torch.allclose(mean_y, y.double().mean(dim=1), rtol=1e-5, atol=1e-5)
    assert torch.allclose(var_y, y.double().var(dim=1, unbiased=False), rtol=1e-4, atol=1e-5)
    Wq, csq, bq = _fold(C, 3 * C, dt, g)
    qkv = torch.empty(M, 3 * C, device="cuda", dtype=dt)
    capi.gemm_ex(y, Wq, qkv, bias=bq, stats_in=st_y, colsum=csq, ln_C=C, ln_eps=1e-6)
    torch.cuda.synchronize()
    _check_consumer(y, st_y, Wq, csq, bq, qkv, False, dt, what="mlp -> qkv parts=%d" % parts)


# --------------------------------------------------------------------------------------------------- engine wiring
@pytest.mark.parametrize("name", ["tiny", "medium", "xlarge"])
def test_engine_layernorm_fold_matches_float64(name):
    """Captures of a real forward (batch 2: the unfused MLP GEMMs): block1's qkv and fc1 against float64 LayerNorm -> linear with
    the checkpoint's own (unfolded) weights on the captured inputs.  Checks the load-time fold (ln_w into W, ln_b into the bias,
    the [q_bias, 0, v_bias] layout)."""
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    cfg = CONFIGS[name]
    C, dt, B = cfg.vit_dim, torch.float16, 2
    sd = synth_state_dict(cfg, 1)
    eng = capi.Engine(cfg, dt)
    eng.load_state_dict(sd)
    T = B * 1600
    caps = {l: eng.capture(l, T * n) for l, n in (("block0", C), ("block1.qkv", 3 * C), ("block1.proj", C), ("block1.fc1", 4 * C))}
    eng.forward(synth_images(B, 0).cuda())
    torch.cuda.synchronize()
    got = eng.capture_results()
    eng.close()
    labels = set(caps)
    assert all(got[l] is not None and got[l].numel() == caps[l].numel() for l in labels), {l: None if got[l] is None else got[l].numel() for l in got}
    p = "backbone.0.encoder.blocks.1."
    w = {k[len(p):]: v.double().cuda() for k, v in sd.items() if k.startswith(p)}
    for inp, outl, norm, lin, bias in (("block0", "block1.qkv", "norm1", "attn.qkv",
                                        torch.cat([w["attn.q_bias"], torch.zeros_like(w["attn.q_bias"]), w["attn.v_bias"]])),
                                       ("block1.proj", "block1.fc1", "norm2", "mlp.fc1", w["mlp.fc1.bias"])):
        x = got[inp].view(T, C).cuda().double()                  # the fp16 values the GEMM read
        y = got[outl].view(T, -1).cuda().double()
        mean, var = x.mean(dim=1, keepdim=True), x.var(dim=1, unbiased=False, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + 1e-6)
        xh = (x - mean) * rstd
        Wt = w[lin + ".weight"]
        Wf = Wt * w[norm + ".weight"]
        pre = xh @ Wf.t() + (bias + Wt @ w[norm + ".bias"])
        gelu = outl.endswith("fc1")
        ref = _gelu64(pre) if gelu else pre
        Wr = Wf.to(dt).double()
        # the weights are stored rounded: |W' - round(W')| <= half an ulp each; plus the bound of the LayerNorm consumer
        e = (xh.abs() @ _half_ulp(Wf, dt).t()) + rstd * (C / 16 * 2.0 ** -22 * (x.abs() @ Wr.abs().t())
                                                        + mean.abs() * Wr.sum(dim=1).abs() * 2.0 ** -21) \
            + (pre.abs() + 1.0) * 2.0 ** -20
        if gelu:
            e = 1.13 * e + 8e-5 * torch.clamp(pre.abs(), min=1.0)
        err = (y - ref).abs()
        bound = e + _half_ulp(ref, dt)
        assert (err <= bound).all(), "%s %s: %d elements out of bound, worst err %.4g" % (name, outl, int((err > bound).sum()), float(err.max()))


# --------------------------------------------------------------------------------------------------- head-major value store
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("heads", [16, 24])
@pytest.mark.parametrize("S", [1600, 6800, 1237])
def test_head_major_store_with_row_zero(dt, heads, S):
    from b200 import capi
    g = _gen(S + heads)
    B, NL = 2, 3
    d = heads * 16
    M = B * S
    A = (torch.randn(M, d, device="cuda", generator=g)).to(dt)
    W = (torch.randn(NL * d, d, device="cuda", generator=g) / d ** 0.5).to(dt)
    bias = torch.randn(NL * d, device="cuda", generator=g)
    flags = (torch.rand(M, device="cuda", generator=g) < 0.15).to(torch.uint8)
    flags[S - 1] = 1                                          # last row of image 0, first of image 1 left unflagged
    flags[S] = 0
    outs = []
    for rz in (flags, torch.zeros_like(flags)):
        out = torch.full((B * NL * heads * S * 16 + 64,), float("nan"), device="cuda", dtype=dt)
        bn, ep, _ = capi.gemm_ex(A, W, out, bias=bias, hm_S=S, hm_heads=heads, hm_slices=NL, row_zero=rz)
        assert ep == "EP_GENERIC"
        outs.append(out)
    torch.cuda.synchronize()
    RAN.add(("EP_GENERIC(head-major)", bn, _dn(dt)))
    for out in outs:
        assert torch.isnan(out[-64:]).all(), "wrote past the value tensor"
    ref = (A.double() @ W.double().t() + bias.double())
    bound = _half_ulp(ref, dt) + d / 16 * 2.0 ** -22 * (A.double().abs() @ W.double().abs().t()) + ref.abs() * 2.0 ** -22
    to_hm = lambda t: t.reshape(B, S, NL, heads, 16).permute(0, 2, 3, 1, 4)
    got, got0 = [o[:-64].view(B, NL, heads, S, 16) for o in outs]
    fl = flags.bool().view(B, S)
    z = got.permute(0, 3, 1, 2, 4)                              # [B, S, NL, heads, 16]
    assert (z[fl] == 0).all(), "flagged rows are not zero"
    assert torch.equal(z[~fl], got0.permute(0, 3, 1, 2, 4)[~fl]), "an unflagged row depends on its neighbours' flags"
    assert ((got0.double() - to_hm(ref)).abs() <= to_hm(bound)).all(), "head-major layout / values"


# --------------------------------------------------------------------------------------------------- LayerNorm variants
def _ln64(x64, w, b, eps):
    mean = x64.mean(dim=1, keepdim=True)
    var = x64.var(dim=1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    return (x64 - mean) * rstd * w.double() + b.double(), mean, rstd


def _ln_bound(x64, ref, w, b, mean, rstd, dt, C):
    """fp32 two-pass LayerNorm: the mean is a sum over a path of at most 8 * chunks + 5 additions (2^-24 each, of at most
    sum|x|); the variance likewise, rsqrtf 2 ulps."""
    path = 8 * math.ceil(C / 256) + 5
    d_mean = path * 2.0 ** -24 * x64.abs().sum(dim=1, keepdim=True) / C
    xh = (x64 - mean) * rstd
    return _half_ulp(ref, dt) + w.double().abs() * (rstd * d_mean + xh.abs() * (path + 4) * 2.0 ** -23) + b.double().abs() * 2.0 ** -23


def _ln_rows(rows, C, dt, g):
    x, _, _ = _kind_rows(rows, C, dt, g)
    return x


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C", [192, 256, 384, 768, 1024])
@pytest.mark.parametrize("where", ["below", "above", "small"])
def test_layernorm_variants_match_float64(dt, C, where):
    from b200 import capi
    thr = 8 * 4 * 2 * _sms()
    rows = {"below": thr - 3, "above": thr + 37, "small": 1001}[where]     # ragged: rows % 4 and rows % 32 != 0
    g = _gen(C * 3 + rows)
    x = _ln_rows(rows, C, dt, g)
    xw = torch.zeros(rows, C + 64, device="cuda", dtype=dt)
    xw[:, :C] = x
    xs = xw[:, :C]
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    b = torch.randn(C, device="cuda", generator=g) * 0.2
    w3 = torch.rand(C, device="cuda", generator=g) + 0.5
    b3 = torch.randn(C, device="cuda", generator=g) * 0.2
    add = (torch.randn(rows, C, device="cuda", generator=g)).to(dt)
    ovr = torch.randn(C, device="cuda", generator=g) * 2 + 0.5
    flag_mod = 97
    flags = (torch.rand(flag_mod, device="cuda", generator=g) < 0.2).to(torch.uint8)
    flags[0] = 1
    eps, eps3 = 1e-5, 1e-2                # different, so that a chained norm using the wrong one shows
    y = torch.full((rows + 3, C), float("nan"), device="cuda", dtype=dt)
    y2 = torch.full((rows, C), float("nan"), device="cuda", dtype=dt)
    y3 = torch.full((rows, C), float("nan"), device="cuda", dtype=dt)
    rpw = capi.layernorm_ex(xs, y, w, b, eps, row_flag=flags, override=ovr, add=add, y2=y2, w3=w3, b3=b3, eps3=eps3, y3=y3)
    torch.cuda.synchronize()
    assert rpw == (4 if rows >= thr and C <= 512 else 1)
    RAN.add(("LN", rpw, C, _dn(dt)))
    assert torch.isnan(y[rows:]).all()
    flagged = flags.bool()[torch.arange(rows, device="cuda") % flag_mod]
    x64 = x.double().clone()
    x64[flagged] = ovr.double()                                     # flagged rows normalise the override vector (fp32)
    ref, mean, rstd = _ln64(x64, w, b, eps)
    bound = _ln_bound(x64, ref, w, b, mean, rstd, dt, C)
    err = (y[:rows].double() - ref).abs()
    assert (err <= bound).all(), "y: %d elements out of bound, worst row %d" % (int((err > bound).sum()), int((err > bound).nonzero()[0, 0]))
    # y2 = y + add in the 16-bit type from the kernel's own rounded y
    assert torch.equal(y2, (y[:rows].float() + add.float()).to(dt)), "y2 is not round(round(y) + add)"
    # y3: exactly what a plain call on the rounded y writes
    y3b = torch.empty(rows, C, device="cuda", dtype=dt)
    capi.layernorm_ex(y[:rows], y3b, w3, b3, eps3)
    torch.cuda.synchronize()
    assert torch.equal(y3, y3b), "chained y3 differs from a separate LayerNorm of y in %d elements" % int((y3 != y3b).sum())
    y64 = y[:rows].double()
    ref3, m3, r3 = _ln64(y64, w3, b3, eps3)
    assert ((y3.double() - ref3).abs() <= _ln_bound(y64, ref3, w3, b3, m3, r3, dt, C)).all(), "y3 against float64"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("rpw_rows", ["above", "below"])
def test_layernorm_group_scatter(dt, rpw_rows):
    """The projector's y_group: level rows (B images x H*W) land at rows b*S + level_start + t of the memory; other rows stay NaN."""
    from b200 import capi
    C = 256
    thr = 8 * 4 * 2 * _sms()
    B, S, start = 3, 8500, 6800
    HW = -(-(thr + 5) // B) if rpw_rows == "above" else 1600 + 3
    S = max(S, start + HW)
    g = _gen(HW)
    rows = B * HW
    x = _ln_rows(rows, C, dt, g)
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    b = torch.randn(C, device="cuda", generator=g) * 0.2
    mem = torch.full((B * S, C), float("nan"), device="cuda", dtype=dt)
    rpw = capi.layernorm_ex(x, mem, w, b, 1e-6, y_group=HW, y_group_stride=S, y_row_off=start)
    torch.cuda.synchronize()
    RAN.add(("LN", rpw, C, _dn(dt)))
    plain = torch.empty(rows, C, device="cuda", dtype=dt)
    capi.layernorm_ex(x, plain, w, b, 1e-6)
    torch.cuda.synchronize()
    m = mem.view(B, S, C)
    assert torch.equal(m[:, start:start + HW].reshape(rows, C), plain), "level rows not at their offset"
    assert torch.isnan(m[:, :start]).all() and torch.isnan(m[:, start + HW:]).all(), "rows of other levels were written"
    ref, mean, rstd = _ln64(x.double(), w, b, 1e-6)
    assert ((plain.double() - ref).abs() <= _ln_bound(x.double(), ref, w, b, mean, rstd, dt, C)).all()


def test_every_instance_is_covered():
    """The plans the device builds for the shapes the tests above launch (dry runs, nothing launched) reach every tile width for
    EP_LN, EP_LN_GELU and EP_RESID with statistics, and every specialisation at every width.  The LayerNorm rows-per-warp
    instances are asserted where they run (test_layernorm_variants_match_float64)."""
    from b200 import capi
    sms = _sms()
    seen = set()

    def plan(M, K, N, **kw):
        A = torch.empty(M, K, device="cuda", dtype=torch.float16)
        W = torch.empty(N, K, device="cuda", dtype=torch.float16)
        out = torch.empty(M, N, device="cuda", dtype=torch.float16)
        bn, ep, _ = capi.gemm_ex(A, W, out, dry_run=True, **kw)
        seen.add((ep, bn))

    cs = torch.zeros(3072, device="cuda")
    for C, N in ((192, 576), (192, 768), (384, 1152), (384, 1536), (768, 2304), (768, 3072), (256, 512)):
        st = torch.zeros(128 * sms + 37, 2, 2, device="cuda")
        for M in (128 * sms + 37, 1000):
            for act in (capi.ACT_NONE, capi.ACT_GELU):
                plan(M, C, N, stats_in=st[:M], colsum=cs, ln_C=C, ln_eps=1e-6, act=act)
    buf = _stats_buf(128 * sms + 37)
    for C, size in PRODUCER_CASES:
        plan(PRODUCER_M[size](), C, C, stats_out=buf)
    for ep in ("EP_LN", "EP_LN_GELU"):
        assert {b for e, b in seen if e == ep} == {64, 128, 192, 256}, seen
    assert {b for e, b in seen if e == "EP_RESID"} == {64, 128, 192, 256}, seen
    for bn, N in SPEC_SHAPES.items():
        M = 128 * 8 + 45 if bn == 64 else 128 * sms + 45
        seen.clear()
        plan(M, 256, N)
        plan(M, 256, N, act=capi.ACT_GELU)
        assert seen == {("EP_BIAS", bn), ("EP_BIAS_ACT", bn)}, seen
