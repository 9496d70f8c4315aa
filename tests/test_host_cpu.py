"""CPU tests of the host side: the C-ABI library loads and exports what include/lwdetr_b200.h declares, the
drop-in module keeps the reference's surface, host helpers match torch, and the N>1 plumbing works on gloo."""
import argparse
import copy
import json
import os
import re
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS, config_from_args  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402


def _args(name):
    import ref_import
    a = ref_import.reference_args(CONFIGS[name])
    a.lr, a.lr_encoder, a.lr_vit_layer_decay, a.lr_component_decay, a.weight_decay = 1e-4, 1.5e-4, 0.8, 0.7, 1e-4
    return a


def test_library_exports_every_declared_symbol():
    with open(os.path.join(ROOT, "include", "lwdetr_b200.h")) as f:
        hdr = f.read()
    declared = set(re.findall(r"LWDETR_API\s+[\w\s\*]+?\b(lwdetr_\w+)\s*\(", hdr))
    assert len(declared) >= 20
    lib = capi.lib()
    for name in declared:
        assert hasattr(lib, name), name
    assert declared == set(capi.exported_symbols())
    assert lib.lwdetr_abi_version() == 1


def test_create_without_gpu_fails_loudly():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        capi.Engine(CONFIGS["tiny"], torch.float16)
    import ctypes
    h = ctypes.c_void_p()
    cs = capi.config_struct(CONFIGS["tiny"])
    assert capi.lib().lwdetr_create(ctypes.byref(cs), 0, ctypes.byref(h)) != 0
    assert b"no CUDA device" in capi.lib().lwdetr_last_error()


def test_host_bicubic_matches_torch():
    g = torch.Generator().manual_seed(0)
    src = torch.randn(14, 14, 7, generator=g)
    for n_out in (40, 14, 9):
        ref = F.interpolate(src.permute(2, 0, 1)[None], size=(n_out, n_out), mode="bicubic", align_corners=False)[0].permute(1, 2, 0)
        assert (capi.host_bicubic(src, n_out) - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("name", ["tiny", "small", "large", "xlarge"])
def test_dropin_module_surface(name):
    from models import build_model
    from models.backbone import Joiner
    a = _args(name)
    model, criterion, post = build_model(a)
    assert a.num_feature_levels == len(a.projector_scale)
    with open(os.path.join(ROOT, "tests", "golden", "state_dict_%s.json" % name)) as f:
        ref = {k: tuple(v) for k, v in json.load(f).items()}
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == ref
    model.load_state_dict(synth_state_dict(CONFIGS[name], 1), strict=True)
    assert isinstance(model.backbone, Joiner)
    pairs = model.backbone[0].get_named_param_lr_pairs(a, prefix="backbone.0")
    assert all(k.startswith("backbone.0.encoder") for k in pairs)
    blk0 = pairs["backbone.0.encoder.blocks.0.attn.qkv.weight"]
    L = a.vit_encoder_num_layers
    assert abs(blk0["lr"] - a.lr_encoder * 0.8 ** L * 0.49) < 1e-12 and blk0["weight_decay"] == a.weight_decay
    assert pairs["backbone.0.encoder.pos_embed"]["weight_decay"] == 0.0
    assert any("transformer.decoder" in n for n, _ in model.named_parameters())
    assert model.transformer.d_model == a.hidden_dim
    assert hasattr(model.backbone[0].encoder.blocks[0], "drop_path")
    model.update_drop_path(0.1, L)
    model.update_dropout(0.0)
    m2 = copy.deepcopy(model)
    assert torch.equal(m2.class_embed.weight, model.class_embed.weight) and m2.class_embed.weight is not model.class_embed.weight
    m2 = m2.half().float().eval()
    assert "bbox" in post and hasattr(criterion, "weight_dict")
    with pytest.raises(RuntimeError, match="CUDA"):
        m2(torch.zeros(1, 3, 640, 640))
    model.train()
    with pytest.raises(RuntimeError, match="inference"):
        model(torch.zeros(1, 3, 640, 640))


def test_config_from_args_rejects_unreleased_variants():
    a = _args("small")
    assert config_from_args(a).vit_dim == 192
    a.encoder = "res18vd"
    with pytest.raises(NotImplementedError):
        config_from_args(a)
    b = _args("small")
    b.two_stage = False
    with pytest.raises(NotImplementedError):
        config_from_args(b)


def test_nested_tensor_contract():
    from util.misc import NestedTensor, nested_tensor_from_tensor_list
    imgs = [torch.ones(3, 4, 6), torch.ones(3, 5, 3)]
    nt = nested_tensor_from_tensor_list(imgs)
    assert isinstance(nt, NestedTensor) and nt.tensors.shape == (2, 3, 5, 6) and nt.mask.shape == (2, 5, 6)
    assert not nt.mask[0, :4, :6].any() and nt.mask[0, 4].all() and nt.mask[1, :, 3:].all()
    t, m = nt.decompose()
    assert t is nt.tensors and m is nt.mask
    same = nested_tensor_from_tensor_list(torch.zeros(2, 3, 8, 8))
    assert not same.mask.any()


def test_postprocess_matches_oracle():
    from models.lwdetr import PostProcess
    from oracle import lwdetr_oracle as orc
    g = torch.Generator().manual_seed(1)
    out = {"pred_logits": torch.randn(2, 300, 91, generator=g), "pred_boxes": torch.rand(2, 300, 4, generator=g)}
    sizes = torch.tensor([[480, 640], [600, 400]])
    a = PostProcess(100)(out, sizes)
    b = orc.postprocess(out, sizes, 100)
    for x, y in zip(a, b):
        for k in ("scores", "labels", "boxes"):
            assert torch.allclose(x[k].float(), y[k].float(), atol=1e-5)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from b200.dist import broadcast_module_weights, shard_range
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg).eval()
    if rank == 0:
        model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    n = broadcast_module_weights(model, src=0)
    ref = synth_state_dict(cfg, 1)
    ok = all(torch.equal(v, ref[k]) for k, v in model.state_dict().items() if v.is_floating_point())
    q.put((rank, ok, n, shard_range(10, rank, world)))
    dist.destroy_process_group()


def test_weight_broadcast_and_sharding_world2_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    assert [r[1] for r in res] == [True, True]
    assert res[0][2] == res[1][2] > 12e6
    assert res[0][3] == (0, 5) and res[1][3] == (5, 10)


def test_bench_clock_sampler_windows_and_reasons():
    """bench.py's nvidia-smi sampler: only samples inside the load window count, idle clocks are dropped from the
    median, throttle reasons are collected, and an empty window reports 'unavailable' instead of inventing numbers."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.ClockSampler(0)
    na = "Not Active"
    s.rows = [
        [10.0, "345", "1965", "120", "0x0", na, na, na, na],            # before the window (idle)
        [20.1, "1965", "1965", "900", "0x4", na, na, na, "Active"],
        [20.2, "1950", "1965", "910", "0x4", na, na, na, "Active"],
        [20.3, "1965", "1965", "905", "0x0", na, na, na, na],
        [20.4, "345", "1965", "130", "0x0", na, na, na, na],            # load already over: dropped as < half of max
        [30.0, "1200", "1965", "500", "0x8", "Active", na, na, na],     # after the window
    ]
    assert s.count_in(20.0, 20.5) == 4
    r = s.summary(20.0, 20.5)
    assert r["sm_mhz"] == 1965.0 and r["sm_max_mhz"] == 1965.0 and r["reasons"] == ["sw_power_cap"] and r["samples"] == 4
    assert s.summary(40.0, 50.0) == {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
    assert "hw_slowdown" in s.summary()["reasons"]
