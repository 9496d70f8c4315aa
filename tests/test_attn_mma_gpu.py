"""The mma.sync attention kernels of attn.cu (attn_short_kernel, attn_kernel with 4 and 8 warps, and their polynomial-exp2
instances) kernel by kernel against float64 softmax attention, through lwdetr_attention_ex, which reports the instance it ran.

Every case lays its buffers out as the decoder does: q and k are column slices of one matrix with a padded row stride, v lies in
a separate matrix with another stride, and out is a column slice of a wider NaN-filled matrix whose other columns must stay
NaN.  A few packed q / k / v cases run the wgmma kernel (attn_wg.cu) under the same bound.

Reference: float64 on the GPU from the same 16-bit q, k, v.  With s_j the raw scores of a query row, p_j = exp(scale (s_j -
max s)) (the largest is 1) and o = sum p_j v_j / sum p_j, every output element must satisfy err <= bound with

  bound = (1 + 2u) sum_j (u_j p_j + a) dev_j / sum p  +  L 2^-23 sum_j p_j |v_j| / sum p  +  2u |o|  +  tiny
  u_j   = u + e_exp + scale (es_j + max_j es_j),   es_j = dh 2^-24 sum_i |q_i k_ji|  (fp32 score error, raw units)

  u      2^-11 (fp16) or 2^-8 (bf16): the rounding of P to the 16-bit MMA operand and of the output;
  e_exp  2^-21 for ex2.approx, 7.5e-5 on the n-tiles whose exponentials take the polynomial (ptx.cuh: exp2_poly2);
  dev_j  |v_j - o|: the mma.sync kernels take the row sums of the same rounded P (an MMA against ones), so a rounding of p_j
         moves o by (v_j - o) times its share.  The wgmma kernel sums the unrounded P: dev_j = |v_j|;
  a      the absolute floor of P: 2^-25 for fp16 (subnormal P against the running maximum), 2^-124 for bf16 (ex2.approx.ftz
         flushes below 2^-126, and the polynomial clamps its argument at 2^-125 of the running maximum);
  L 2^-23  the fp32 accumulation of P V over L keys;  tiny  the smallest 16-bit subnormal.

Run as a script, the file is the child that runs the polynomial instances (LWDETR_B200_ATTN_POLY is read once per process):
  python tests/test_attn_mma_gpu.py run      -> JSON {"ratios": {instance: max err/bound}, "failures": [...]}
  python tests/test_attn_mma_gpu.py dry-run  -> JSON list of the instances every case would reach (no device needed)."""
import json
import os
import subprocess
import sys
from collections import namedtuple

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "lw-detr_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

pytestmark = pytest.mark.gpu

DTYPES = ("float16", "bfloat16")
POLY_MASK = {0: 0, 1: 0x24, 2: 0x49}
BUDGET = 1 << 26                # float64 elements of the largest [rows, L, dh] reference tensor

Case = namedtuple("Case", "seqlen nseq heads dh kind scale packed")


def _case(seqlen, nseq, heads, dh, kind="random", scale=None, packed=False):
    return Case(seqlen, nseq, heads, dh, kind, scale, packed)


SHORT_L = (1, 7, 16, 63, 64, 65, 100, 104, 105, 111, 112)       # attn_short_kernel: one chunk, the 40- and 48-key tails
LONG4_L = (113, 128, 129, 300, 511, 1023)                      # attn_kernel, 4 warps
LONG8_L = (1024, 1025, 1600, 2049)                             # attn_kernel, 8 warps


def _cases():
    cs = []
    for dh in (16, 32, 64):
        cs += [_case(L, 3, 1, dh) for L in SHORT_L]            # 3 items: fewer than the resident CTAs
        cs += [_case(L, 2, 3, dh) for L in LONG4_L]
        cs += [_case(L, 2, 2, dh) for L in LONG8_L]
        for kind in ("late", "onehot", "wide", "bigv", "seam"):
            cs += [_case(L, 3, 2, dh, kind) for L in (105, 112, 129, 1023, 1025)]
        cs += [_case(L, 3, 2, dh, "seam") for L in (7, 64, 100)]
    # 7680 items: the persistent walk and its 3-deep prefetch ring wrap many times
    cs += [_case(100, 640, 12, 16), _case(105, 640, 12, 32)]
    # the decoder's own shapes: 300 queries x 8 heads (small / medium), x 12 heads (large / xlarge), 100 x 8 (tiny)
    for B in (1, 2, 64):
        cs += [_case(300, B, 8, 32), _case(300, B, 12, 32), _case(100, B, 8, 32)]
    cs += [_case(300, 2, 4, 32, scale=0.3), _case(100, 3, 4, 16, scale=0.9)]
    # the wgmma kernel: windows, global, the 40-key tail, a late maximum
    cs += [_case(100, 8, 4, 32, packed=True), _case(1600, 1, 4, 16, packed=True), _case(104, 4, 4, 64, packed=True),
           _case(1600, 2, 2, 32, "late", packed=True)]
    return cs


CASES = _cases()


def _id(c):
    return "%s-L%d-n%d-h%d-dh%d%s%s" % (c.kind, c.seqlen, c.nseq, c.heads, c.dh, "" if c.scale is None else "-s%g" % c.scale,
                                        "-packed" if c.packed else "")


def expected(c, policy):
    """The instance the dispatch rule of include/lwdetr_b200.h names for a case."""
    if c.packed:
        return ("wg", 0, 0)
    if c.seqlen <= 112:
        return ("mma_short", 0, POLY_MASK[policy] if c.dh != 64 else 0)
    warps = 8 if c.seqlen >= 1024 else 4
    return ("mma", warps, POLY_MASK[policy] if warps == 8 and c.dh != 64 else 0)


def takes_poly(c):
    return not c.packed and c.dh != 64 and (c.seqlen <= 112 or c.seqlen >= 1024)


def _strides(c):
    """Row strides (elements) of the qk / qkv matrix, the v matrix and the out matrix, and the column offsets of v and out."""
    C = c.heads * c.dh
    return (3 * C + 8 if c.packed else 2 * C + 8), C + 24, 8, C + 40, 8


def dry_run_instances(policy):
    """(dtype, kernel, dh, warps, mask) every case reaches, from integer addresses laid out like the real buffers."""
    import torch
    from b200 import capi
    out = []
    for c in CASES:
        C = c.heads * c.dh
        ldqk, ldv, voff, ldo, ooff = _strides(c)
        base, vbase, obase = 1 << 32, 1 << 36, 1 << 38
        q = (base, ldqk)
        k = (base + 2 * C, ldqk)
        v = (base + 4 * C, ldqk) if c.packed else (vbase + 2 * voff, ldv)
        o = (obase + 2 * ooff, ldo)
        for dt in DTYPES:
            r = capi.attention_ex(q, k, v, o, c.nseq, c.seqlen, c.heads, c.dh, c.dh ** -0.5, dry_run=True, dtype=getattr(torch, dt))
            got = (r["kernel"], r["warps"], r["poly_mask"])
            assert got == expected(c, policy), (_id(c), got, expected(c, policy))
            out.append((dt, r["kernel"], c.dh, r["warps"], r["poly_mask"]))
    return sorted(set(out))


# ------------------------------------------------------------------------------------------------------------- inputs
def _inputs(c, dt, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    C, L, n = c.heads * c.dh, c.seqlen, c.nseq * c.seqlen
    q = torch.randn(n, C, device="cuda", generator=g)
    k = torch.randn(n, C, device="cuda", generator=g)
    v = torch.randn(n, C, device="cuda", generator=g)
    pos = torch.arange(n, device="cuda") % L
    if c.kind == "random":
        q, k = q * 1.5, k * 1.5
    elif c.kind == "late":
        # keys that dwarf everything before them arrive in later chunks: the running maximum moves up to three times
        for frac, gain in ((0.35, 4.0), (0.6, 10.0), (0.9, 25.0)):
            j = int(frac * L)
            k[(pos >= j) & (pos < j + 3)] *= gain
    elif c.kind == "onehot":
        # one key overwhelms the rest (P one-hot): o is that key's value row
        q = 1.0 + 0.1 * q
        k = 0.5 * k
        k[pos == (2 * L) // 3] = 30.0
    elif c.kind == "wide":
        # scores spread over more than 150 in log2 units: most P underflow, the polynomial's clamp is reached
        q, k = q * 7.0, k * 7.0
    elif c.kind == "bigv":
        v = (v * 1e4).clamp(-3e4, 3e4)
    elif c.kind == "seam":
        # sequences end to end: the first rows of every sequence carry dominant keys whose values alternate in sign from one
        # sequence to the next, so a key read past the end of a sequence moves its output far outside the bound
        q = 1.0 + 0.2 * q
        first = pos < 8
        k[first] = 6.0
        sign = 1.0 - 2.0 * ((torch.arange(n, device="cuda") // L) % 2).float()
        v[first] = (100.0 * sign[first]).unsqueeze(1)
        k[pos == L - 3] = 6.5
    tdt = getattr(torch, dt)
    return q.to(tdt), k.to(tdt), v.to(tdt)


# ---------------------------------------------------------------------------------------------------------- reference
def check_against_float64(out, q, k, v, nseq, L, heads, dh, scale, mask, wg_form):
    """Asserts err <= bound (module docstring) at every element of out [nseq*L, heads*dh]; returns max(err / bound)."""
    import torch
    bf = q.dtype == torch.bfloat16
    u = 2.0 ** -8 if bf else 2.0 ** -11
    a = 2.0 ** -124 if bf else 2.0 ** -25
    tiny = 2.0 ** -133 if bf else 2.0 ** -24

    def heads_major(t):
        return t.double().reshape(nseq, L, heads, dh).transpose(1, 2).reshape(nseq * heads, L, dh)
    Q, K, V, O = heads_major(q), heads_major(k), heads_major(v), heads_major(out)
    j = torch.arange(L, device=q.device)
    e_exp = torch.where(((mask >> ((j % 64) // 8)) & 1).bool(), 7.5e-5, 2.0 ** -21).double()
    G = nseq * heads
    gc = max(1, min(G, BUDGET // (L * L * dh)))
    rc = max(1, min(L, BUDGET // (gc * L * dh)))
    worst = 0.0
    for g0 in range(0, G, gc):
        Kc, Vc = K[g0:g0 + gc], V[g0:g0 + gc]
        Kabs, Vabs = Kc.abs(), Vc.abs()
        for r0 in range(0, L, rc):
            Qc, Oc = Q[g0:g0 + gc, r0:r0 + rc], O[g0:g0 + gc, r0:r0 + rc]
            s = Qc @ Kc.transpose(1, 2)
            es = dh * 2.0 ** -24 * (Qc.abs() @ Kabs.transpose(1, 2))
            p = torch.exp(scale * (s - s.amax(-1, keepdim=True)))
            sp = p.sum(-1, keepdim=True)
            o = (p @ Vc) / sp
            uj = u + e_exp + scale * (es + es.amax(-1, keepdim=True))
            w = uj * p + a
            if wg_form:
                t1 = (w @ Vabs) / sp
            else:
                dev = (Vc.unsqueeze(1) - o.unsqueeze(2)).abs_()          # [g, rows, L, dh]
                t1 = torch.einsum("gqk,gqkd->gqd", w, dev) / sp
                del dev
            bound = (1 + 2 * u) * t1 + L * 2.0 ** -23 * (p @ Vabs) / sp + 2 * u * o.abs() + tiny
            err = (Oc - o).abs()
            bad = ~(err <= bound)                                         # NaN output fails too
            if bad.any():
                i = bad.nonzero()[0].tolist()
                raise AssertionError("element (seq*head %d, row %d, col %d): got %r, float64 %r, bound %.3e" % (
                    g0 + i[0], r0 + i[1], i[2], Oc[tuple(i)].item(), o[tuple(i)].item(), bound[tuple(i)].item()))
            worst = max(worst, (err / bound).max().item())
    return worst


def run_case(c, dt, policy):
    """Runs one case on the device; returns (instance, max err/bound)."""
    import torch
    from b200 import capi
    tdt = getattr(torch, dt)
    C, n = c.heads * c.dh, c.nseq * c.seqlen
    ldqk, ldv, voff, ldo, ooff = _strides(c)
    q, k, v = _inputs(c, dt, seed=c.seqlen * 131 + c.dh * 7 + c.nseq + len(c.kind))
    buf = torch.zeros(n, ldqk, device="cuda", dtype=tdt)
    buf[:, :C], buf[:, C:2 * C] = q, k
    qv, kv = buf[:, :C], buf[:, C:2 * C]
    if c.packed:
        buf[:, 2 * C:3 * C] = v
        vv = buf[:, 2 * C:3 * C]
    else:
        vbuf = torch.zeros(n, ldv, device="cuda", dtype=tdt)
        vbuf[:, voff:voff + C] = v
        vv = vbuf[:, voff:voff + C]
    obuf = torch.full((n, ldo), float("nan"), device="cuda", dtype=tdt)
    ov = obuf[:, ooff:ooff + C]
    scale = c.dh ** -0.5 if c.scale is None else c.scale
    r = capi.attention_ex(qv, kv, vv, ov, c.nseq, c.seqlen, c.heads, c.dh, scale)
    got = (r["kernel"], r["warps"], r["poly_mask"])
    assert got == expected(c, policy), (got, expected(c, policy))
    torch.cuda.synchronize()
    assert torch.isnan(obuf[:, :ooff]).all() and torch.isnan(obuf[:, ooff + C:]).all(), "columns outside out were written"
    # the kernel computes with scale * log2(e) rounded to fp32; the reference uses the scale that product stands for
    scale_eff = float(torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)) / 1.4426950408889634
    ratio = check_against_float64(ov, qv, kv, vv, c.nseq, c.seqlen, c.heads, c.dh, scale_eff, r["poly_mask"], c.packed)
    return (dt, r["kernel"], c.dh, r["warps"], r["poly_mask"]), ratio


# ---------------------------------------------------------------------------------------------------------- the tests
RATIOS = {}


def _note(inst, ratio):
    RATIOS[inst] = max(RATIOS.get(inst, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    cm = request.config.pluginmanager.get_plugin("capturemanager")
    if tr is None or cm is None or not RATIOS:
        return
    with cm.global_and_fixture_disabled():
        tr.write_line("")
        for (dt, kern, dh, warps, mask), r in sorted(RATIOS.items()):
            tr.write_line("attention %-9s %-9s dh %2d warps %d mask 0x%02x: max err/bound %.3f" % (kern, dt, dh, warps, mask, r))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", CASES, ids=_id)
def test_attention_within_float64_bound(c, dt):
    if os.environ.get("LWDETR_B200_ATTN_POLY", "0") not in ("", "0"):
        pytest.skip("runs the default instances; the polynomial ones run in test_polynomial_instances")
    inst, ratio = run_case(c, dt, 0)
    _note(inst, ratio)


@pytest.mark.parametrize("policy", [1, 2])
def test_polynomial_instances(policy):
    """The polynomial-exp2 instances: the cases that reach them, in a child process with LWDETR_B200_ATTN_POLY = policy."""
    env = dict(os.environ, LWDETR_B200_ATTN_POLY=str(policy))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "run"], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for key, ratio in res["ratios"].items():
        _note(tuple(json.loads(key)), ratio)
    assert not res["failures"], res["failures"][:10]
    assert any(json.loads(key)[4] == POLY_MASK[policy] for key in res["ratios"])


def _child(mode):
    policy = int(os.environ.get("LWDETR_B200_ATTN_POLY", "0") or 0)
    if mode == "dry-run":
        print(json.dumps(dry_run_instances(policy)))
        return
    ratios, failures = {}, []
    for c in CASES:
        if not takes_poly(c):
            continue
        for dt in DTYPES:
            try:
                inst, ratio = run_case(c, dt, policy)
                key = json.dumps(list(inst))
                ratios[key] = max(ratios.get(key, 0.0), ratio)
            except AssertionError as e:
                failures.append("%s/%s: %s" % (_id(c), dt, e))
    print(json.dumps({"ratios": ratios, "failures": failures}))


if __name__ == "__main__":
    _child(sys.argv[1] if len(sys.argv) > 1 else "run")
