"""The fused ViT MLP of the 192-wide encoder (mlp.cu vit_mlp_kernel) on the GPU: the kernel against a float64 restatement,
the engine schedule that uses it (tiny, small, from 11 images of 640x640 on) or not (medium, batch 1), and CUDA-graph replay
of a forward that runs it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

C, HID = 192, 768
DTYPES = [torch.float16, torch.bfloat16]


def _partials(x64, parts):
    """Per-row LayerNorm partials (sum, M2) over `parts` equal column slices, as the statistics producers write them."""
    xs = x64.view(x64.shape[0], parts, -1)
    s = xs.sum(dim=2)
    m2 = ((xs - xs.mean(dim=2, keepdim=True)) ** 2).sum(dim=2)
    return torch.stack([s, m2], dim=2).float().contiguous()


def _gelu64(v):
    return 0.5 * v * (1.0 + torch.erf(v / 2 ** 0.5))


def _inputs(M, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(M, C, device="cuda", generator=g) * 0.8 + 0.3).to(dt)
    x[min(5, M - 1)] = (1000.0 + 0.25 * torch.randn(C, device="cuda", generator=g)).to(dt)   # mean 1000, spread 0.25
    W1 = (torch.randn(HID, C, device="cuda", generator=g) / C ** 0.5).to(dt)
    W2 = (torch.randn(C, HID, device="cuda", generator=g) / HID ** 0.5).to(dt)
    b1 = torch.randn(HID, device="cuda", generator=g) * 0.5
    cs1 = W1.double().sum(dim=1).float()
    b2 = torch.randn(C, device="cuda", generator=g) * 0.1
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    return x, W1, W2, b1, cs1, b2, gamma


def _reference(x, W1, W2, b1, cs1, b2, gamma, dt, eps=1e-6):
    """LN -> fc1 -> GELU -> round to the compute dtype -> fc2 -> gamma * y + residual, in float64."""
    x64 = x.double()
    mean = x64.mean(dim=1, keepdim=True)
    rstd = 1.0 / torch.sqrt(x64.var(dim=1, unbiased=False, keepdim=True) + eps)
    h = _gelu64(rstd * (x64 @ W1.double().t()) - rstd * mean * cs1.double() + b1.double())
    h = h.to(dt).double()
    return x64 + gamma.double() * (h @ W2.double().t() + b2.double())


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("M", [1600, 51200, 1600 * 3 + 37])
def test_vit_mlp_kernel_matches_float64(dt, M):
    from b200 import capi
    x, W1, W2, b1, cs1, b2, gamma = _inputs(M, dt, M)
    parts_in = 6 if M == 1600 else 2
    stats_in = _partials(x.double(), parts_in)
    wide = torch.full((M, 3 * C), float("nan"), device="cuda", dtype=dt)
    out = wide[:, C:2 * C]                                          # ld_out = 576 != C
    parts_out = 2 if M != 1600 else 6
    stats_out = torch.full((M, parts_out, 2), float("nan"), device="cuda", dtype=torch.float32)
    capi.vit_mlp(x, stats_in, W1, cs1, b1, W2, b2=b2, gamma=gamma, out=out, stats_out=stats_out)
    torch.cuda.synchronize()
    assert torch.isnan(wide[:, :C]).all() and torch.isnan(wide[:, 2 * C:]).all(), "wrote outside its columns"
    ref = _reference(x, W1, W2, b1, cs1, b2, gamma, dt)
    # the residual (up to 1000 in one row) dominates the scale: judge the MLP branch y - x on its own scale
    got_d = out.double() - x.double()
    ref_d = ref - x.double()
    scale = ref_d.abs().max().item()
    err = (got_d - ref_d).abs().max().item()
    ulp_x = x.double().abs().max(dim=1).values * (2.0 ** -10 if dt == torch.float16 else 2.0 ** -7)
    bound = (4e-3 if dt == torch.float16 else 2.5e-2) * scale
    rows_err = (got_d - ref_d).abs().max(dim=1).values
    assert (rows_err <= bound + ulp_x).all(), "max err %.4g vs scale %.4g" % (err, scale)
    normal = torch.ones(M, dtype=torch.bool, device="cuda")
    normal[min(5, M - 1)] = False
    rel = ((got_d - ref_d)[normal].norm() / ref_d[normal].norm()).item()
    assert rel <= (6e-3 if dt == torch.float16 else 3e-2), "rel-L2 %.3g" % rel
    # the emitted partials combine to the float64 mean / variance of the rounded output rows
    o64 = out.double()
    st = stats_out.double()
    n_p = C / parts_out
    mean = st[:, :, 0].sum(dim=1) / C
    var = (st[:, :, 1].sum(dim=1) + n_p * ((st[:, :, 0] / n_p - mean[:, None]) ** 2).sum(dim=1)) / C
    assert torch.allclose(mean, o64.mean(dim=1), rtol=1e-5, atol=1e-5)
    assert torch.allclose(var, o64.var(dim=1, unbiased=False), rtol=1e-4, atol=1e-5)


def _ops(name, dt, fuse=1, batch=16):
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    cfg = CONFIGS[name]
    eng = capi.Engine(cfg, dt)
    eng.set_option("fuse_layernorm", fuse)
    eng.load_state_dict(synth_state_dict(cfg, 1))
    eng.forward(synth_images(batch, 0).cuda())
    labels = [o[0] for o in eng.ops()]
    eng.close()
    return cfg, labels


@pytest.mark.parametrize("name", ["tiny", "small"])
@pytest.mark.parametrize("dt", DTYPES)
def test_schedule_fuses_the_mlp_of_the_192_wide_encoder(name, dt):
    cfg, labels = _ops(name, dt)
    assert not any(l.endswith(".fc1") for l in labels)
    for i in range(cfg.vit_depth):
        assert labels.count("block%d" % i) == 1


def test_schedule_keeps_the_two_gemms_elsewhere():
    _, labels = _ops("medium", torch.float16)
    assert "block0.fc1" in labels and "block0" in labels
    _, labels = _ops("small", torch.float16, fuse=0)
    assert "block0.fc1" in labels and "block0" in labels
    _, labels = _ops("small", torch.float16, batch=1)              # 13 tiles of 128 rows: the GEMMs fill more SMs
    assert "block0.fc1" in labels and "block0" in labels


def test_cuda_graph_replay_is_bit_identical_to_eager():
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    cfg = CONFIGS["small"]
    eng = capi.Engine(cfg, torch.float16)
    eng.load_state_dict(synth_state_dict(cfg, 1))
    xs = [synth_images(16, s).cuda() for s in (0, 1)]             # 200 tiles: the fused path
    eager = [{k: v.clone() for k, v in eng.forward(x).items() if k.startswith("pred")} for x in xs]
    eng.set_option("cuda_graph", 1)
    for _ in range(2):
        for x, ref in zip(xs, eager):
            out = eng.forward(x)
            torch.cuda.synchronize()
            assert torch.equal(out["pred_logits"], ref["pred_logits"]) and torch.equal(out["pred_boxes"], ref["pred_boxes"])
    eng.close()
