"""ctypes binding of include/lwdetr_b200.h.

Every function signature and struct layout is read from the header when this module loads, so the header is the only
description of the ABI; a form the reader does not know is an error.  The shared library is built in-tree by
tools/build.py (``__graft_entry__.build()``).  There is no fallback: if the header or the library is missing or a call
fails, a RuntimeError is raised.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "liblwdetr_b200.so")

F16, BF16, F16_E4M3 = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU = 0, 1, 2, 3

_lib = None

_vp = ctypes.c_void_p
HEADER_PATH = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "include", "lwdetr_b200.h")
_SCALARS = {"int": ctypes.c_int, "int8_t": ctypes.c_int8, "int16_t": ctypes.c_int16, "int32_t": ctypes.c_int32,
            "int64_t": ctypes.c_int64, "uint8_t": ctypes.c_uint8, "uint32_t": ctypes.c_uint32, "float": ctypes.c_float,
            "double": ctypes.c_double}


def _unreadable(decl, where):
    raise RuntimeError("lwdetr_b200: cannot read `%s` (%s) in include/lwdetr_b200.h" % (" ".join(decl.split()), where))


def _ctype(decl, where, field=False):
    """(name, ctypes type) of one declaration of the header: a parameter, a return type (no name) or a struct field.
    Pointers and array parameters are c_void_p, except a lone char* (a C string); a field array is a ctypes array."""
    m = re.fullmatch(r"\s*(?:const\s+)?(\w+)\s*((?:\*\s*(?:const\b\s*)?)*)(\w*)\s*(?:\[(\d+)\])?\s*", decl)
    if m and not (m.group(2) and m.group(4)):
        base, stars, name, n = m.group(1), m.group(2).count("*"), m.group(3), m.group(4)
        if stars or (n and not field):
            return name, ctypes.c_char_p if (base, stars) == ("char", 1) else _vp
        if base in _SCALARS:
            return name, _SCALARS[base] * int(n) if n else _SCALARS[base]
        if base == "void" and not name and not field:
            return name, None
    _unreadable(decl, where)


def _read_header(path):
    """The C ABI as the header declares it: ({function: (restype, argtypes)}, {struct typedef name: ctypes.Structure}).
    It reads the header's own forms only: `LWDETR_API <ret> lwdetr_x(<args>);` and `typedef struct { ... } lwdetr_y;` of
    scalars, pointers and fixed arrays (and opaque `typedef struct x x;` handles); anything else there is an error."""
    if not os.path.exists(path):
        raise RuntimeError("lwdetr_b200: %s not found - the C ABI is read from it (there is no copy of it in Python)" % path)
    with open(path) as f:
        src = re.sub(r"^\s*#.*$", " ", re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S), flags=re.M)
    structs = {}
    for decl in re.findall(r"\btypedef\b[^;{]*(?:\{[^}]*\})?[^;]*;", src):
        m = re.fullmatch(r"typedef\s+struct\s*\{([^}]*)\}\s*(\w+)\s*;", decl)
        if m is None:
            if not re.fullmatch(r"typedef\s+struct\s+(\w+)\s+\1\s*;", decl):
                _unreadable(decl, "typedef")
            continue
        fields = []
        for stmt in filter(str.strip, m.group(1).split(";")):
            t = re.match(r"\s*(?:const\s+)?\w+", stmt) or _unreadable(stmt, m.group(2))
            fields += [_ctype(t.group(0) + " " + d, m.group(2), True) for d in stmt[t.end():].split(",")]
        structs[m.group(2)] = type(m.group(2), (ctypes.Structure,), {"_fields_": fields})
    sigs = {}
    for decl in re.findall(r"\bLWDETR_API\b[^;]*;", src):
        m = re.fullmatch(r"LWDETR_API\s+([^;(]*?)\s*\b(lwdetr_\w+)\s*\(([^()]*)\)\s*;", decl) or _unreadable(decl, "prototype")
        args = [] if m.group(3).strip() == "void" else [_ctype(a, m.group(2))[1] for a in m.group(3).split(",")]
        sigs[m.group(2)] = (_ctype(m.group(1), m.group(2))[1], args)
    return sigs, structs


_SIGNATURES, _STRUCTS = _read_header(HEADER_PATH)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "lwdetr_b200: %s not found - run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback)" % LIB_PATH)
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: %s" % (what, lib().lwdetr_last_error().decode()))


def ptr(t):
    """Device/host address of a torch tensor (or None)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def dtype_code(torch_dtype):
    """Engine compute mode of a torch dtype: float16, bfloat16, or float8_e4m3fn for the fp16 engine whose encoder qkv / fc1
    GEMMs run in e4m3 (LWDETR_F16_E4M3)."""
    import torch
    if torch_dtype == torch.float16:
        return F16
    if torch_dtype == torch.bfloat16:
        return BF16
    if torch_dtype == torch.float8_e4m3fn:
        return F16_E4M3
    raise RuntimeError("lwdetr_b200 computes in float16, bfloat16 or float8_e4m3fn (e4m3 encoder mode), got %s" % torch_dtype)


def kernel_dtype_code(torch_dtype):
    """dtype code of the 16-bit kernel-level entry points (tensors in float16 or bfloat16 only)."""
    code = dtype_code(torch_dtype)
    if code not in (F16, BF16):
        raise RuntimeError("lwdetr_b200 kernels take float16 or bfloat16 tensors, got %s" % torch_dtype)
    return code


def io_dtype(torch_dtype):
    """The 16-bit type of an engine's activations (and of 16-bit images it takes): float16 in the e4m3 mode."""
    import torch
    return torch.float16 if torch_dtype == torch.float8_e4m3fn else torch_dtype


def _addr(t):
    """Address of a tensor for a pointer field of a ctypes.Structure (None: NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr(device=None):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def gemm(A, W, out, bias=None, gamma=None, resid=None, resid_mod=0, act=ACT_NONE, M=None, K=None, N=None,
         rows_in=0, remap_rows=0, shuffle_cout=0, IH=0, IW=0):
    """out = epilogue(A @ W.T); A [M, K] (row stride A.stride(0)), W [N, K] contiguous."""
    import torch
    M = A.shape[0] if M is None else M
    K = A.shape[1] if K is None else K
    N = W.shape[0] if N is None else N
    check(lib().lwdetr_gemm(kernel_dtype_code(A.dtype), ptr(A), A.stride(0), M, K, ptr(W), N, ptr(bias), ptr(gamma),
                            ptr(resid), 0 if resid is None else resid.stride(0), resid_mod, act, ptr(out),
                            out.stride(0), 1 if out.dtype == torch.float32 else 0, rows_in, remap_rows,
                            shuffle_cout, IH, IW, stream_ptr()), "lwdetr_gemm")
    return out


EP_NAMES = {0: "EP_GENERIC", 1: "EP_BIAS", 2: "EP_BIAS_ACT", 3: "EP_LN", 4: "EP_LN_GELU", 5: "EP_RESID"}


GemmArgs = _STRUCTS["lwdetr_gemm_args"]


def gemm_ex(A, W, out, bias=None, gamma=None, resid=None, resid_mod=0, act=ACT_NONE, M=None, K=None, N=None,
            stats_in=None, colsum=None, ln_C=0, ln_eps=0.0, stats_out=None, hm_S=0, hm_heads=0, hm_slices=0, row_zero=None,
            dry_run=False):
    """lwdetr_gemm_ex: lwdetr_gemm plus the LayerNorm consumer (stats_in fp32 [M, parts, 2] contiguous, colsum fp32 [N], ln_C,
    ln_eps), the statistics producer (stats_out fp32 [M, >= parts_out, 2] contiguous), the head-major store (hm_S, hm_heads,
    hm_slices; out a contiguous buffer) and row_zero (uint8 [M]).  Returns (bn, epilogue name, stats_parts_out) of the plan
    that ran (dry_run: was built, nothing launched)."""
    import torch
    a = GemmArgs()
    a.dtype = kernel_dtype_code(A.dtype)
    a.A, a.lda, a.M, a.K = A.data_ptr(), A.stride(0), A.shape[0] if M is None else M, A.shape[1] if K is None else K
    a.W, a.N = W.data_ptr(), W.shape[0] if N is None else N
    a.bias, a.gamma = _addr(bias), _addr(gamma)
    a.resid, a.ld_resid, a.resid_mod = _addr(resid), 0 if resid is None else resid.stride(0), resid_mod
    a.act, a.out, a.out_fp32 = act, out.data_ptr(), 1 if out.dtype == torch.float32 else 0
    a.ld_out = 16 if hm_S else out.stride(0)
    if stats_in is not None:
        a.stats_in, a.stats_parts_in = stats_in.data_ptr(), stats_in.shape[1]
    a.colsum, a.ln_C, a.ln_eps = _addr(colsum), ln_C, float(ln_eps)
    if stats_out is not None:
        a.stats_out = stats_out.data_ptr()
    a.hm_S, a.hm_heads, a.hm_slices, a.row_zero = hm_S, hm_heads, hm_slices, _addr(row_zero)
    a.dry_run = 1 if dry_run else 0
    check(lib().lwdetr_gemm_ex(ctypes.byref(a), stream_ptr()), "lwdetr_gemm_ex")
    return a.bn, EP_NAMES[a.epilogue], a.stats_parts_out


LayerNormArgs = _STRUCTS["lwdetr_layernorm_args"]


def layernorm_ex(x, y, w, b, eps, rows=None, C=None, row_flag=None, override=None, add=None, y2=None,
                 y_group=0, y_group_stride=0, y_row_off=0, w3=None, b3=None, eps3=0.0, y3=None):
    """lwdetr_layernorm_ex: y = LN(x) with the optional row flag (uint8 [flag_mod]) + override vector, y2 = y + add, y_group
    row scatter and chained y3 = LN(y; w3, b3, eps3).  2-D tensors with any row stride.  Returns the rows per warp that ran."""
    a = LayerNormArgs()
    a.x, a.ldx, a.y, a.ldy = x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0)
    a.w, a.b, a.eps = _addr(w), _addr(b), float(eps)
    a.rows, a.C = x.shape[0] if rows is None else rows, x.shape[1] if C is None else C
    if row_flag is not None:
        a.row_flag, a.flag_mod, a.override_vec = row_flag.data_ptr(), row_flag.numel(), _addr(override)
    if y2 is not None:
        a.add_src, a.ld_add, a.y2, a.ldy2 = add.data_ptr(), add.stride(0), y2.data_ptr(), y2.stride(0)
    a.y_group, a.y_group_stride, a.y_row_off = y_group, y_group_stride, y_row_off
    if y3 is not None:
        a.w3, a.b3, a.eps3, a.y3, a.ldy3 = _addr(w3), _addr(b3), float(eps3), y3.data_ptr(), y3.stride(0)
    check(lib().lwdetr_layernorm_ex(kernel_dtype_code(x.dtype), ctypes.byref(a), stream_ptr()), "lwdetr_layernorm_ex")
    return a.rows_per_warp


def conv3x3(X, Wk, out, B, OH, OW, stride, Cin, bias=None, act=ACT_NONE):
    """X NHWC [B, s*OH, s*OW, ldx] (uses channels [0, Cin)), Wk [N, 9*Cin], out [B*OH*OW, ld_out]."""
    check(lib().lwdetr_conv3x3(kernel_dtype_code(X.dtype), ptr(X), X.stride(2), B, OH, OW, stride, Cin, ptr(Wk),
                               Wk.shape[0], ptr(bias), act, ptr(out), out.stride(0), stream_ptr()),
          "lwdetr_conv3x3")
    return out


def layernorm(x, y, w, b, eps, rows=None, C=None):
    rows = x.shape[0] if rows is None else rows
    C = x.shape[1] if C is None else C
    check(lib().lwdetr_layernorm(kernel_dtype_code(x.dtype), ptr(x), x.stride(0), ptr(y), y.stride(0), ptr(w), ptr(b), eps,
                                 rows, C, stream_ptr()), "lwdetr_layernorm")
    return y


def attention(q, k, v, out, nseq, seqlen, heads, dh, scale):
    """q/k/v/out: 2-D views [nseq*seqlen, heads*dh] (any row stride)."""
    check(lib().lwdetr_attention(kernel_dtype_code(q.dtype), ptr(q), q.stride(0), ptr(k), k.stride(0), ptr(v), v.stride(0),
                                 ptr(out), out.stride(0), nseq, seqlen, heads, dh, scale, stream_ptr()),
          "lwdetr_attention")
    return out


ATTN_KERNELS = {0: "wg", 1: "mma", 2: "mma_short"}


AttentionArgs = _STRUCTS["lwdetr_attention_args"]


def attention_ex(q, k, v, out, nseq, seqlen, heads, dh, scale, dry_run=False, dtype=None):
    """lwdetr_attention_ex.  q / k / v / out: 2-D views [nseq*seqlen, heads*dh] (any row stride), or (address, leading
    dimension) pairs of integers, which a dry run never dereferences (dtype then names the torch dtype).  Returns
    {"kernel": "wg" | "mma" | "mma_short", "warps": 4 | 8 | 0, "poly_mask": 0 | 0x24 | 0x49} of the kernel that ran (dry_run:
    would run; nothing is launched and no CUDA call is made)."""
    def mat(t):
        return t if isinstance(t, tuple) else (t.data_ptr(), t.stride(0))
    a = AttentionArgs()
    a.dtype = kernel_dtype_code(q.dtype if dtype is None else dtype)
    (a.q, a.ldq), (a.k, a.ldk), (a.v, a.ldv), (a.out, a.ldo) = mat(q), mat(k), mat(v), mat(out)
    a.nseq, a.seqlen, a.heads, a.dh, a.scale, a.dry_run = nseq, seqlen, heads, dh, float(scale), 1 if dry_run else 0
    check(lib().lwdetr_attention_ex(ctypes.byref(a), None if dry_run else stream_ptr()), "lwdetr_attention_ex")
    return {"kernel": ATTN_KERNELS[a.kernel], "warps": a.warps, "poly_mask": a.poly_mask}


def value_to_head_major(value, B, S, M):
    """[B*S, M*16] token-major (view, any row stride) -> contiguous head-major [B, M, S, 16] (what value_proj's epilogue writes)."""
    return value.reshape(B, S, M, 16).permute(0, 2, 1, 3).contiguous()


def _level_table(shapes):
    """HOST int32 arrays (spatial shapes [L, 2], level starts [L]) of consecutive levels of the given (H, W)."""
    starts, acc = [], 0
    for h, w in shapes:
        starts.append(acc)
        acc += h * w
    return (ctypes.c_int32 * (2 * len(shapes)))(*[v for hw in shapes for v in hw]), (ctypes.c_int32 * len(shapes))(*starts)


MSDA_MAX_BANDS = 16


def msda_plan(shapes, S=None):
    """lwdetr_msda_plan (no device): the bands msda_forward streams for consecutive levels of the given (H, W), S = their
    token count unless given.  A list of (level, row0, own0, own1, tok0, bytes); empty: the direct-gather kernel runs."""
    sh, st = _level_table(shapes)
    S = sum(h * w for h, w in shapes) if S is None else S
    nb = ctypes.c_int32()
    rows = (ctypes.c_int32 * (6 * MSDA_MAX_BANDS))()
    check(lib().lwdetr_msda_plan(len(shapes), ctypes.cast(sh, _vp), ctypes.cast(st, _vp), S, ctypes.byref(nb), ctypes.cast(rows, _vp)),
          "lwdetr_msda_plan")
    return [tuple(rows[6 * k:6 * k + 6]) for k in range(nb.value)]


def conv3x3_plan(OH, OW):
    """lwdetr_conv3x3_plan (no device): the (TW, TH) output tile of the implicit-GEMM 3x3 convolution over an OH x OW grid."""
    tw, th = ctypes.c_int32(), ctypes.c_int32()
    check(lib().lwdetr_conv3x3_plan(OH, OW, ctypes.byref(tw), ctypes.byref(th)), "lwdetr_conv3x3_plan")
    return tw.value, th.value


def msda_forward(value_hm, offs_logits, ref, out, B, S, Lq, M, L, P, shapes, valid_ratio=None, v_image_stride=None):
    """value_hm head-major [B, M, S, 16], offs_logits [B*Lq, 3*M*L*P], ref fp32 [B*Lq, 4], out [B*Lq, M*16]."""
    sh, st = _level_table(shapes)
    stride = M * S * 16 if v_image_stride is None else v_image_stride
    check(lib().lwdetr_msda_forward(kernel_dtype_code(value_hm.dtype), ptr(value_hm), stride, ptr(offs_logits),
                                    offs_logits.stride(0), ptr(ref), ptr(valid_ratio), ptr(out), out.stride(0), B, S, Lq, M, L, P,
                                    ctypes.cast(sh, _vp), ctypes.cast(st, _vp), stream_ptr()), "lwdetr_msda_forward")
    return out


ET_F32, ET_F16, ET_BF16 = 0, 1, 2
_ET_OF = {"float32": ET_F32, "float16": ET_F16, "bfloat16": ET_BF16}


def _et_code(dtype, what):
    """LWDETR_ET_* of a float32, float16 or bfloat16 dtype; else RuntimeError "<what> must be float32, float16 or ..."."""
    code = _ET_OF.get(str(dtype).replace("torch.", ""))
    if code is None:
        raise RuntimeError("%s must be float32, float16 or bfloat16, got %s" % (what, dtype))
    return code


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step=64):
    """The reference operator (ms_deform_attn_func.py:28-38 -> MSDA.ms_deform_attn_forward): value [B,S,M,D],
    spatial_shapes int64 [L,2], level_start_index int64 [L], sampling_loc [B,Lq,M,L,P,2], attn_weight [B,Lq,M,L,P], all
    CUDA and contiguous; returns [B, Lq, M*D] in value's dtype (fp32, fp16 or bf16)."""
    import torch
    et = _et_code(value.dtype, "ms_deform_attn_forward: value")
    for name, t in (("value", value), ("spatial_shapes", spatial_shapes), ("level_start_index", level_start_index),
                    ("sampling_loc", sampling_loc), ("attn_weight", attn_weight)):
        if not t.is_cuda:
            raise RuntimeError("ms_deform_attn_forward: %s must be a CUDA tensor (Not implemented on the CPU)" % name)   # ms_deform_attn.h:34
        if not t.is_contiguous():
            raise RuntimeError("ms_deform_attn_forward: %s tensor has to be contiguous" % name)                          # ms_deform_attn_cuda.cu:28-32
    if sampling_loc.dtype != value.dtype or attn_weight.dtype != value.dtype:
        raise RuntimeError("ms_deform_attn_forward: value, sampling_loc and attn_weight must share one dtype")
    if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
        raise RuntimeError("ms_deform_attn_forward: spatial_shapes / level_start_index must be int64")
    B, S, M, D = value.shape
    Lq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    out = torch.empty(B, Lq, M * D, device=value.device, dtype=value.dtype)
    check(lib().lwdetr_ms_deform_attn_forward(et, ptr(value), ptr(spatial_shapes), ptr(level_start_index), ptr(sampling_loc),
                                              ptr(attn_weight), ptr(out), B, S, M, D, Lq, L, P, int(im2col_step), stream_ptr()),
          "lwdetr_ms_deform_attn_forward")
    return out


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step=64):
    """MSDA.ms_deform_attn_backward (ms_deform_attn.h:37-60): fp32 CUDA tensors -> (grad_value, grad_sampling_loc, grad_attn_weight)."""
    import torch
    for name, t in (("value", value), ("sampling_loc", sampling_loc), ("attn_weight", attn_weight), ("grad_output", grad_output)):
        if not t.is_cuda:
            raise RuntimeError("ms_deform_attn_backward: %s must be a CUDA tensor (Not implemented on the CPU)" % name)
        if t.dtype != torch.float32:
            raise RuntimeError("ms_deform_attn_backward: %s must be float32" % name)
        if not t.is_contiguous():
            raise RuntimeError("ms_deform_attn_backward: %s tensor has to be contiguous" % name)
    B, S, M, D = value.shape
    Lq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    gv, gl, ga = torch.empty_like(value), torch.empty_like(sampling_loc), torch.empty_like(attn_weight)
    check(lib().lwdetr_ms_deform_attn_backward(ptr(value), ptr(spatial_shapes), ptr(level_start_index), ptr(sampling_loc), ptr(attn_weight),
                                               ptr(grad_output), ptr(gv), ptr(gl), ptr(ga), B, S, M, D, Lq, L, P, int(im2col_step),
                                               stream_ptr()), "lwdetr_ms_deform_attn_backward")
    return gv, gl, ga


def topk(score, k):
    import torch
    B, S = score.shape
    idx = torch.empty(B, k, device=score.device, dtype=torch.int32)
    check(lib().lwdetr_topk(ptr(score), B, S, k, ptr(idx), stream_ptr()), "lwdetr_topk")
    return idx


def _detector_outputs(pred_logits, pred_boxes, target_sizes):
    """What postprocess() and query_best() read: (B, nq, num_classes, logits, boxes, target sizes), contiguous fp32 on the
    logits' device."""
    import torch
    B, nq, ncls = pred_logits.shape
    logits = pred_logits.float().contiguous()
    boxes = pred_boxes.float().contiguous()
    return B, nq, ncls, logits, boxes, target_sizes.to(device=logits.device, dtype=torch.float32).contiguous()


def postprocess(pred_logits, pred_boxes, target_sizes, num_select):
    """Fused PostProcess (lwdetr.py:515-544) on CUDA fp32 tensors -> (scores [B,k] fp32, labels [B,k] int32, boxes [B,k,4] fp32)."""
    import torch
    B, nq, ncls, logits, boxes, ts = _detector_outputs(pred_logits, pred_boxes, target_sizes)
    parts = (nq * ncls + 16383) // 16384
    work = torch.empty(B * parts * num_select, device=logits.device, dtype=torch.int32)
    scores = torch.empty(B, num_select, device=logits.device, dtype=torch.float32)
    labels = torch.empty(B, num_select, device=logits.device, dtype=torch.int32)
    out = torch.empty(B, num_select, 4, device=logits.device, dtype=torch.float32)
    check(lib().lwdetr_postprocess(ptr(logits), ptr(boxes), ptr(ts), B, nq, ncls, num_select, ptr(work), ptr(scores), ptr(labels),
                                   ptr(out), stream_ptr()), "lwdetr_postprocess")
    return scores, labels, out


TILE_METRICS = {"iou": 0, "ios": 1}     # LWDETR_TILE_IOU / LWDETR_TILE_IOS


TileViewStruct = _STRUCTS["lwdetr_tile_view"]


def tile_merge(scores, labels, boxes, views, num_frames, score_threshold=0.0, iou_threshold=0.5, metric="ios", max_det=300):
    """lwdetr_tile_merge: the per-view output of postprocess() (scores fp32 [V, k], labels int32 [V, k], xyxy boxes fp32
    [V, k, 4] in each view's crop pixels, CUDA) and the views as (frame, x0, y0) triples (frames non-decreasing) -> per frame
    the first max_det survivors of a class-aware greedy NMS over all its views, in frame pixels: (scores fp32 [F, max_det],
    labels int32 [F, max_det], boxes fp32 [F, max_det, 4], counts int32 [F]), unused slots score 0, label -1, zero box.
    metric: "ios" (intersection over the smaller box) or "iou".  Stream-ordered, no synchronisation."""
    import torch
    if metric not in TILE_METRICS:
        raise RuntimeError("tile_merge: metric must be one of %s, got %r" % (", ".join(TILE_METRICS), metric))
    V, k = scores.shape
    if tuple(labels.shape) != (V, k) or tuple(boxes.shape) != (V, k, 4) or len(views) != V:
        raise RuntimeError("tile_merge: scores %s, labels %s, boxes %s and %d views do not describe one [V, k] set"
                           % (tuple(scores.shape), tuple(labels.shape), tuple(boxes.shape), len(views)))
    if scores.dtype != torch.float32 or labels.dtype != torch.int32 or boxes.dtype != torch.float32:
        raise RuntimeError("tile_merge: scores / boxes must be float32 and labels int32")
    scores, labels, boxes = scores.contiguous(), labels.contiguous(), boxes.contiguous()
    arr = (TileViewStruct * V)(*[TileViewStruct(int(f), int(x0), int(y0)) for f, x0, y0 in views])
    F, dev = int(num_frames), scores.device
    out_s = torch.empty(F, max_det, device=dev, dtype=torch.float32)
    out_l = torch.empty(F, max_det, device=dev, dtype=torch.int32)
    out_b = torch.empty(F, max_det, 4, device=dev, dtype=torch.float32)
    counts = torch.empty(F, device=dev, dtype=torch.int32)
    check(lib().lwdetr_tile_merge(ptr(scores), ptr(labels), ptr(boxes), V, k, ctypes.cast(arr, _vp), F, float(score_threshold),
                                  float(iou_threshold), TILE_METRICS[metric], int(max_det), ptr(out_s), ptr(out_l), ptr(out_b),
                                  ptr(counts), stream_ptr(dev)), "lwdetr_tile_merge")
    return out_s, out_l, out_b, counts


def query_best(pred_logits, pred_boxes, target_sizes):
    """lwdetr_query_best: one detection per query, its best class (CUDA fp32 tensors as for postprocess) -> (scores fp32
    [B, nq], labels int32 [B, nq], boxes fp32 [B, nq, 4]), each entry with the bits postprocess() gives that (query, class)
    pair."""
    import torch
    B, nq, ncls, logits, boxes, ts = _detector_outputs(pred_logits, pred_boxes, target_sizes)
    dev = logits.device
    scores = torch.empty(B, nq, device=dev, dtype=torch.float32)
    labels = torch.empty(B, nq, device=dev, dtype=torch.int32)
    out = torch.empty(B, nq, 4, device=dev, dtype=torch.float32)
    check(lib().lwdetr_query_best(ptr(logits), ptr(boxes), ptr(ts), B, nq, ncls, ptr(scores), ptr(labels), ptr(out), stream_ptr(dev)),
          "lwdetr_query_best")
    return scores, labels, out


TrackParams = _STRUCTS["lwdetr_track_params"]
TrackRecord = _STRUCTS["lwdetr_track_record"]
ReidParams = _STRUCTS["lwdetr_reid_params"]


def _track_outputs(B, m, dev):
    """The outputs of one tracker step on dev: ids int32 [B, m], scores fp32, labels int32, boxes fp32 [B, m, 4], index
    int32 and counts int32 [B], in the C calls' order."""
    import torch
    return (torch.empty(B, m, device=dev, dtype=torch.int32), torch.empty(B, m, device=dev, dtype=torch.float32),
            torch.empty(B, m, device=dev, dtype=torch.int32), torch.empty(B, m, 4, device=dev, dtype=torch.float32),
            torch.empty(B, m, device=dev, dtype=torch.int32), torch.empty(B, device=dev, dtype=torch.int32))


def _motion(motion, B, dev, what):
    """The camera motion of B frames as contiguous float64 [B, 4] on dev, or None."""
    import torch
    if motion is None:
        return None
    if tuple(motion.shape) != (B, 4):
        raise RuntimeError("%s: motion must be [%d, 4], got %s" % (what, B, tuple(motion.shape)))
    return motion.to(device=dev, dtype=torch.float64).contiguous()


class _DeviceObject:
    """What Tracker, MotionEstimator and Zones share: a C object made on one device from a parameter struct (its handle in _t),
    reset per stream and destroyed by close()."""

    RESET = DESTROY = None                               # the subclass's C calls

    def __init__(self, num_streams, device, create, *params):
        import torch
        self.num_streams = int(num_streams)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._t = _vp()
        with torch.cuda.device(self.device):
            check(getattr(lib(), create)(self.num_streams, *[ctypes.byref(p) for p in params], ctypes.byref(self._t)), create)

    def _params(self, struct, default, params):
        """struct from the C call `default`, then the keyword arguments; a name struct lacks is an error."""
        p = struct()
        getattr(lib(), default)(ctypes.byref(p))
        bad = set(params) - {n for n, _ in struct._fields_}
        if bad:
            raise RuntimeError("%s: unknown parameters %s" % (type(self).__name__, ", ".join(sorted(bad))))
        for n, v in params.items():
            setattr(p, n, v)
        return p

    def close(self):
        if self._t:
            getattr(lib(), self.DESTROY)(self._t)
            self._t = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _ids(ids):
        ids = [int(x) for x in ids]
        return (ctypes.c_int32 * max(len(ids), 1))(*ids), len(ids)

    def _stream_ids(self, ids, B, what):
        """The HOST int32 array of the stream ids of B frames (default range(B)); RuntimeError naming `what` unless B are given."""
        arr, n = self._ids(range(B) if ids is None else ids)
        if n != B:
            raise RuntimeError("%s: %d stream ids for %d frames" % (what, n, B))
        return arr

    def reset(self, streams):
        """The streams start again (stream-ordered): a tracker's at frame 1 and id 1 with empty lists, an estimator's at
        their next frame, a zones object's at frame 1 with no records and zero counters (geometry kept)."""
        arr, n = self._ids(streams)
        check(getattr(lib(), self.RESET)(self._t, ctypes.cast(arr, _vp), n, stream_ptr(self.device)), self.RESET)


class Tracker(_DeviceObject):
    """ByteTrack on the device for num_streams camera streams (lwdetr_tracker_*, the contract in include/lwdetr_b200.h).
    Parameters are lwdetr_track_params' fields, ByteTrack's defaults unless given; new_track_thresh defaults to
    track_thresh + 0.1.  With embedding_dim (lwdetr_reid_params: embedding_dim, proximity_thresh, appearance_thresh,
    ema_alpha; BoT-SORT's defaults unless given) the tracker also associates by appearance (BoT-SORT's re-identification
    cost, lwdetr_track_reid); update() then takes embeddings.  All calls of one tracker must run on one CUDA stream (the
    current one at each call)."""

    REID = ("embedding_dim", "proximity_thresh", "appearance_thresh", "ema_alpha")
    RESET, DESTROY = "lwdetr_tracker_reset", "lwdetr_tracker_destroy"

    def __init__(self, num_streams, device=None, **params):
        reid = {n: params.pop(n) for n in self.REID if n in params and params[n] is not None}
        for n in self.REID:
            params.pop(n, None)
        if reid and "embedding_dim" not in reid:
            raise RuntimeError("Tracker: %s given without embedding_dim" % ", ".join(sorted(reid)))
        if params.get("new_track_thresh") is None:
            params["new_track_thresh"] = params.get("track_thresh", 0.5) + 0.1
        self.params = self._params(TrackParams, "lwdetr_track_params_default", params)
        self.reid = self._params(ReidParams, "lwdetr_reid_params_default", reid) if reid else None
        self.embedding_dim = int(self.reid.embedding_dim) if reid else None
        if reid:
            super().__init__(num_streams, device, "lwdetr_tracker_create_reid", self.params, self.reid)
        else:
            super().__init__(num_streams, device, "lwdetr_tracker_create", self.params)
        # frames each stream has had since create or reset, counted on the host by update() and BoxFlow.propagate() (the
        # keyframe schedule of LWDETR.track(detect_every=)); a replayed CUDA graph of those calls, or a direct C call on this
        # tracker, advances the device's frame counter without it
        self.frames = [0] * self.num_streams

    def reset(self, streams):
        super().reset(streams)
        for s in streams:
            self.frames[int(s)] = 0

    def update(self, scores, labels, boxes, stream_ids=None, max_out=None, motion=None, embeddings=None):
        """One frame for each of B distinct streams: scores fp32 [B, k], labels int [B, k], xyxy boxes fp32 [B, k, 4] (CUDA;
        stream_ids default range(B)) -> (ids int32 [B, max_out], scores fp32, labels int32, boxes fp32 [B, max_out, 4], index
        int32 (the entry of each track), counts int32 [B]); unused slots id 0, score 0, label -1, zero box, index -1.
        max_out defaults to k.  motion: float64 [B, 4] camera motion of each frame (MotionEstimator.estimate), which warps
        every track of the stream after the predict (lwdetr_track_ex); None tracks as for a still camera.
        embeddings (a tracker with embedding_dim D only): CUDA [B, k, D] float32, float16 or bfloat16, any row stride (the
        last dimension contiguous), the appearance of each entry (lwdetr_track_reid); None: no entry has appearance, which
        gives ByteTrack's result.  Stream-ordered, no synchronisation."""
        import torch
        B, k = scores.shape
        if tuple(labels.shape) != (B, k) or tuple(boxes.shape) != (B, k, 4):
            raise RuntimeError("Tracker.update: scores %s, labels %s and boxes %s do not describe one [B, k] set"
                               % (tuple(scores.shape), tuple(labels.shape), tuple(boxes.shape)))
        dev = self.device
        scores = scores.to(device=dev, dtype=torch.float32).contiguous()
        labels = labels.to(device=dev, dtype=torch.int32).contiguous()
        boxes = boxes.to(device=dev, dtype=torch.float32).contiguous()
        ids = self._stream_ids(stream_ids, B, "Tracker.update")
        m = k if max_out is None else int(max_out)
        out = _track_outputs(B, m, dev)
        motion = _motion(motion, B, dev, "Tracker.update")
        if self.reid is not None:
            code, ld = ET_F32, 0
            if embeddings is not None:
                D = self.embedding_dim
                if tuple(embeddings.shape) != (B, k, D):
                    raise RuntimeError("Tracker.update: embeddings must be [%d, %d, %d], got %s" % (B, k, D, tuple(embeddings.shape)))
                if embeddings.device != dev:
                    raise RuntimeError("Tracker.update: embeddings are on %s but the tracker lives on %s" % (embeddings.device, dev))
                code = _et_code(embeddings.dtype, "Tracker.update: embeddings")
                if embeddings.stride(2) != 1 or embeddings.stride(0) != k * embeddings.stride(1):
                    embeddings = embeddings.contiguous()
                ld = embeddings.stride(1)
            check(lib().lwdetr_track_reid(self._t, ptr(scores), ptr(labels), ptr(boxes), ptr(motion), ptr(embeddings), code, ld, B, k,
                                          ctypes.cast(ids, _vp), m, *map(ptr, out), stream_ptr(dev)), "lwdetr_track_reid")
            self._last_embeddings = embeddings      # keep alive until the stream has consumed it
        elif embeddings is not None:
            raise RuntimeError("Tracker.update: embeddings need a tracker made with embedding_dim")
        elif motion is None:
            check(lib().lwdetr_track(self._t, ptr(scores), ptr(labels), ptr(boxes), B, k, ctypes.cast(ids, _vp), m, *map(ptr, out),
                                     stream_ptr(dev)), "lwdetr_track")
        else:
            check(lib().lwdetr_track_ex(self._t, ptr(scores), ptr(labels), ptr(boxes), ptr(motion), B, k, ctypes.cast(ids, _vp), m,
                                        *map(ptr, out), stream_ptr(dev)), "lwdetr_track_ex")
        self._advance(ids, B)
        return out

    def _advance(self, ids, n):
        for i in range(n):
            self.frames[ids[i]] += 1

    def export(self, stream_id):
        """Synchronous: (records, (frame, next_id, overflow)) of one stream, records a list of dicts in list order (tracked,
        then lost) with id, state (1 tracked, 2 lost), activated, start, end, score, label, index, mean (8 float64: cx, cy, a,
        h, then velocities) and cov (12 float64: P, C, V per coordinate)."""
        import numpy as np
        cap = int(self.params.capacity)
        arr = (TrackRecord * cap)()
        cnt = ctypes.c_int32()
        fno = (ctypes.c_int32 * 3)()
        check(lib().lwdetr_tracker_export(self._t, int(stream_id), ctypes.cast(arr, _vp), cap, ctypes.byref(cnt), ctypes.cast(fno, _vp)),
              "lwdetr_tracker_export")
        recs = [dict(id=r.id, state=r.state, activated=r.activated, start=r.start_frame, end=r.end_frame, score=np.float32(r.score),
                     label=r.label, index=r.index, mean=np.array(r.mean[:], np.float64), cov=np.array(r.cov[:], np.float64))
                for r in arr[:min(cnt.value, cap)]]
        return recs, tuple(fno)

    def export_embeddings(self, stream_id):
        """Synchronous, a tracker with embedding_dim D only: (embeddings float32 [n, D], has bool [n]) of one stream's
        records in export()'s order; a row is valid where has is True (the track has an embedding)."""
        import numpy as np
        if self.reid is None:
            raise RuntimeError("Tracker.export_embeddings: the tracker was made without embedding_dim")
        cap, D = int(self.params.capacity), self.embedding_dim
        emb = np.zeros((cap, D), np.float32)
        has = np.zeros(cap, np.int8)
        cnt = ctypes.c_int32()
        check(lib().lwdetr_tracker_export_embeddings(self._t, int(stream_id), emb.ctypes.data_as(_vp), cap, ctypes.byref(cnt),
                                                     has.ctypes.data_as(_vp)), "lwdetr_tracker_export_embeddings")
        n = min(cnt.value, cap)
        return emb[:n], has[:n].astype(bool)


GmcParams = _STRUCTS["lwdetr_gmc_params"]


GMC_OK, GMC_FIRST_FRAME, GMC_SIZE_CHANGED, GMC_FEW_POINTS, GMC_FEW_INLIERS = 0, 1, 2, 3, 4


class MotionEstimator(_DeviceObject):
    """Camera motion per video stream on the device (lwdetr_gmc_*, the contract in include/lwdetr_b200.h): the similarity
    from each stream's previous frame to its current one, for Tracker.update(motion=...).  Parameters are
    lwdetr_gmc_params' fields (defaults: lwdetr_gmc_params_default; max_height / max_width bound the frames and size the
    device table).  All calls of one estimator must run on one CUDA stream (the current one at each call)."""

    RESET, DESTROY = "lwdetr_gmc_reset", "lwdetr_gmc_destroy"

    def __init__(self, num_streams, device=None, **params):
        self.params = self._params(GmcParams, "lwdetr_gmc_params_default", params)
        super().__init__(num_streams, device, "lwdetr_gmc_create", self.params)

    def estimate(self, frames, streams=None):
        """One frame for each of B distinct streams (capi.Frames, or frames as Frames takes them; an NV12 frame is read
        through its luma plane only, so its colorspace does not matter) -> (motion float64 [B, 4] (a, b, tx, ty): x' = a x -
        b y + tx, y' = b x + a y + ty from the stream's previous frame to this one in frame pixels; status int32 [B]
        (GMC_*); inliers int32 [B]).  streams defaults to range(B).  Stream-ordered, no synchronisation."""
        return self._call("estimate", frames, streams)

    def observe(self, frames, streams=None):
        """estimate() without the motion (lwdetr_gmc_observe): the streams' pyramids and corners only, so that the next
        estimate() or a BoxFlow on the next frame has this one as its previous frame.  Stream-ordered, no synchronisation."""
        self._call("observe", frames, streams)

    def _call(self, what, frames, streams):
        """lwdetr_gmc_<what>(_nv12) on one frame per stream; the outputs of an estimate, () for an observe."""
        import torch
        if not isinstance(frames, Frames):
            nv12 = isinstance(frames, torch.Tensor) and frames.dim() == 3 and frames.shape[2] != 3
            nv12 = nv12 or (not isinstance(frames, torch.Tensor) and len(frames) > 0 and _is_nv12(frames[0]))
            frames = Frames(frames, self.device, "bt601" if nv12 else None)
        B, dev = len(frames.items), self.device
        ids = self._stream_ids(streams, B, "MotionEstimator." + what)
        out = () if what == "observe" else (torch.empty(B, 4, device=dev, dtype=torch.float64), torch.empty(B, device=dev, dtype=torch.int32),
                                           torch.empty(B, device=dev, dtype=torch.int32))
        name = "lwdetr_gmc_%s%s" % (what, "_nv12" if frames.nv12 else "")
        check(getattr(lib(), name)(self._t, frames.descs(frames.sizes), B, ctypes.cast(ids, _vp), *map(ptr, out), stream_ptr(dev)), name)
        return out

    def export(self, stream_id):
        """Synchronous, waiting for this estimator's last estimate() or reset() and for nothing else on the device: one
        stream's state after its last frame (lwdetr_gmc_export) as a dict: levels (list of uint8 [h_l, w_l] arrays), corners
        float32 [n, 2] (level-0 x, y), flow float32 [m, 4] and found bool [m] (the last call's Lucas-Kanade of the previous
        frame's m corners), valid, size."""
        import numpy as np
        p = self.params
        cap = (p.max_height // p.downscale + 1) * (p.max_width // p.downscale + 1) * 2
        lv = np.zeros(cap, np.uint8)
        corners = np.zeros((p.max_points, 2), np.float32)
        flow = np.zeros((p.max_points, 4), np.float32)
        found = np.zeros(p.max_points, np.int8)
        info = (ctypes.c_int32 * 6)()
        check(lib().lwdetr_gmc_export(self._t, int(stream_id), lv.ctypes.data_as(_vp), cap, corners.ctypes.data_as(_vp),
                                      flow.ctypes.data_as(_vp), found.ctypes.data_as(_vp), ctypes.cast(info, _vp)), "lwdetr_gmc_export")
        valid, h, w, nlev, nc, nf = list(info)
        levels, o = [], 0
        lh, lw = h // p.downscale, w // p.downscale
        for _ in range(nlev + 1):
            levels.append(lv[o:o + lh * lw].reshape(lh, lw).copy())
            o += lh * lw
            lh, lw = (lh + 1) // 2, (lw + 1) // 2
        return dict(valid=bool(valid), size=(h, w), levels=levels, corners=corners[:nc].copy(), flow=flow[:nf].copy(),
                    found=found[:nf].astype(bool))


FlowParams = _STRUCTS["lwdetr_flow_params"]


FLOW_OK, FLOW_FEW_POINTS, FLOW_FB, FLOW_SCALE, FLOW_SMALL, FLOW_SKIPPED, FLOW_NO_PREVIOUS = range(7)


class BoxFlow(_DeviceObject):
    """Per-object optical flow for the frames between detections (the Median Flow tracker, lwdetr_flow_* and
    lwdetr_track_flow in include/lwdetr_b200.h), bound to one MotionEstimator whose pyramids it reads (the estimator must
    have seen each stream's previous frame and its current one, through estimate() or observe()).  Parameters are
    lwdetr_flow_params' fields (defaults: lwdetr_flow_params_default).  Calls must run on the estimator's CUDA stream."""

    DESTROY = "lwdetr_flow_destroy"

    def __init__(self, estimator, **params):
        import torch
        self.params = self._params(FlowParams, "lwdetr_flow_params_default", params)
        self.estimator = estimator                  # kept alive: the flow reads its tables
        self.num_streams = estimator.num_streams
        self.device = estimator.device
        self._t = _vp()
        with torch.cuda.device(self.device):
            check(lib().lwdetr_flow_create(estimator._t, ctypes.byref(self.params), ctypes.byref(self._t)), "lwdetr_flow_create")

    def reset(self, streams):
        raise RuntimeError("BoxFlow.reset: a flow keeps no per-stream state; reset the tracker and the estimator")

    def propagate(self, tracker, streams, motion=None, max_out=None):
        """One flow frame for each listed stream (lwdetr_track_flow): the tracker's confirmed tracks move by their measured
        flow or go Lost, with no detections.  motion: float64 [B, 4] of these frames (MotionEstimator.estimate) or None.
        Returns Tracker.update's tuple; index is -1 for every track.  Stream-ordered, no synchronisation."""
        ids, B = self._ids(streams)
        dev = self.device
        m = int(tracker.params.capacity) if max_out is None else int(max_out)
        out = _track_outputs(B, m, dev)
        motion = _motion(motion, B, dev, "BoxFlow.propagate")
        check(lib().lwdetr_track_flow(tracker._t, self._t, ptr(motion), B, ctypes.cast(ids, _vp), m, *map(ptr, out), stream_ptr(dev)),
              "lwdetr_track_flow")
        tracker._advance(ids, B)
        return out

    def export(self, stream_id):
        """Synchronous: one stream's last flow (lwdetr_flow_export) as a dict of numpy arrays: found (tracks listed), grid,
        per measured track [n, grid^2, ...] seeds, fwd, bwd (level-0 float32 x, y), valid, fb, ncc; per track status, dx, dy,
        s and z (the measurement cx, cy, a, h)."""
        import numpy as np
        T, g2 = int(self.params.max_tracks), int(self.params.grid) ** 2
        seeds, fwd, bwd = (np.zeros((T, g2, 2), np.float32) for _ in range(3))
        valid = np.zeros((T, g2), np.int8)
        fb, ncc = np.zeros((T, g2)), np.zeros((T, g2))
        status = np.zeros(T, np.int32)
        meas = np.zeros((T, 8))
        info = (ctypes.c_int32 * 3)()
        arrs = [seeds, fwd, bwd, valid, fb, ncc, status, meas]
        check(lib().lwdetr_flow_export(self._t, int(stream_id), T, *[a.ctypes.data_as(_vp) for a in arrs], ctypes.cast(info, _vp)),
              "lwdetr_flow_export")
        n = info[1]
        return dict(found=info[0], grid=info[2], seeds=seeds[:n], fwd=fwd[:n], bwd=bwd[:n], valid=valid[:n].astype(bool), fb=fb[:n],
                    ncc=ncc[:n], status=status[:n], dx=meas[:n, 0], dy=meas[:n, 1], s=meas[:n, 2], z=meas[:n, 3:7])


ZonesParams = _STRUCTS["lwdetr_zones_params"]


ZoneRecord = _STRUCTS["lwdetr_zone_record"]


ANCHORS = ("top_left", "top_center", "top_right", "center_left", "center", "center_right", "bottom_left", "bottom_center",
           "bottom_right")
ZONE_LINE_IN, ZONE_LINE_OUT, ZONE_ENTER, ZONE_EXIT, ZONE_FORGET = 1, 2, 3, 4, 5


def zone_geometry(lines=(), polygons=()):
    """One stream's geometry checked against lwdetr_zones_set's rules without any device call: (lines float64 [L, 4],
    polygon sizes int32 [Z], vertices float64 [V, 2]).  Up to 32 lines (ax, ay, bx, by) of non-zero length, up to 32
    polygons of 3 to 256 (x, y) vertices and 2048 vertices in all, every coordinate finite; else ValueError."""
    import numpy as np
    lines = [tuple(float(v) for v in l) for l in lines]
    if len(lines) > 32:
        raise ValueError("Zones.set: at most 32 lines, got %d" % len(lines))
    for i, l in enumerate(lines):
        if len(l) != 4:
            raise ValueError("Zones.set: line %d must be (ax, ay, bx, by), got %d numbers" % (i, len(l)))
        if not all(np.isfinite(l)):
            raise ValueError("Zones.set: line %d has a non-finite coordinate" % i)
        if l[0] == l[2] and l[1] == l[3]:
            raise ValueError("Zones.set: line %d has zero length" % i)
    polys = [np.asarray(p, np.float64) for p in polygons]
    if len(polys) > 32:
        raise ValueError("Zones.set: at most 32 polygons, got %d" % len(polys))
    for i, p in enumerate(polys):
        if p.ndim != 2 or p.shape[1] != 2 or not 3 <= len(p) <= 256:
            raise ValueError("Zones.set: polygon %d must be 3 to 256 (x, y) vertices, got shape %s" % (i, p.shape))
        if not np.isfinite(p).all():
            raise ValueError("Zones.set: polygon %d has a non-finite coordinate" % i)
    sizes = np.array([len(p) for p in polys], np.int32)
    if sizes.sum() > 2048:
        raise ValueError("Zones.set: at most 2048 vertices per stream, got %d" % sizes.sum())
    verts = np.ascontiguousarray(np.concatenate(polys) if polys else np.zeros((0, 2)), np.float64)
    return np.array(lines, np.float64).reshape(-1, 4), sizes, verts


class Zones(_DeviceObject):
    """Line crossings and zone occupancy per camera stream on the device (lwdetr_zones_*, the contract in
    include/lwdetr_b200.h, restated in tools/zone_spec.py): supervision's LineZone / PolygonZone, fed by Tracker.update.
    Parameters are lwdetr_zones_params' fields: num_classes (default 91), capacity (records per stream, default 1024),
    forget_after (frames, default 30), zone_anchor (an anchor index or a name of ANCHORS, default "bottom_center") and
    line_anchors (a bit mask or a list of anchors, default the four corners).  Zones are fixed in frame pixels, also when the
    tracker follows a moving camera.  All calls of one object must run on one CUDA stream (the current one at each call)."""

    RESET, DESTROY = "lwdetr_zones_reset", "lwdetr_zones_destroy"

    def __init__(self, num_streams, device=None, **params):
        if isinstance(params.get("zone_anchor"), str):
            params["zone_anchor"] = ANCHORS.index(params["zone_anchor"])
        la = params.get("line_anchors")
        if la is not None and not isinstance(la, int):
            params["line_anchors"] = sum(1 << (ANCHORS.index(a) if isinstance(a, str) else int(a)) for a in set(la))
        self.params = self._params(ZonesParams, "lwdetr_zones_params_default", params)
        super().__init__(num_streams, device, "lwdetr_zones_create", self.params)

    def set(self, stream, lines=(), polygons=()):
        """Replaces one stream's geometry (frame pixels; zone_geometry's rules, checked before any device call) and clears
        its records and counters.  Synchronous: waits for this object's last launch only.  Not during a stream capture."""
        stream = int(stream)
        if not 0 <= stream < self.num_streams:
            raise ValueError("Zones.set: stream %d outside [0, %d)" % (stream, self.num_streams))
        ln, sizes, verts = zone_geometry(lines, polygons)
        check(lib().lwdetr_zones_set(self._t, stream, ln.ctypes.data_as(_vp), len(ln), sizes.ctypes.data_as(_vp), len(sizes),
                                     verts.ctypes.data_as(_vp)), "lwdetr_zones_set")

    def update(self, ids, labels, boxes, counts, stream_ids=None, max_events=1024):
        """One frame for each of B distinct streams, on Tracker.update's outputs as they are: ids int32 [B, max_out], labels
        [B, max_out], xyxy boxes fp32 [B, max_out, 4], counts [B] (CUDA; stream_ids default range(B)) -> (inside int32 [B,
        max_out]: the bits of each track's uint32 zone mask; occupancy int32 [B, 32]; events int32 [B, max_events, 5] rows
        (id, kind, index, label, dwell), kind ZONE_*, the frame's first max_events in order, unused rows zero; event_counts
        int32 [B], the true number).  Stream-ordered, no synchronisation; graph-safe."""
        import torch
        B, m = ids.shape
        if tuple(labels.shape) != (B, m) or tuple(boxes.shape) != (B, m, 4) or tuple(counts.shape) != (B,):
            raise RuntimeError("Zones.update: ids %s, labels %s, boxes %s and counts %s do not describe one [B, max_out] set"
                               % (tuple(ids.shape), tuple(labels.shape), tuple(boxes.shape), tuple(counts.shape)))
        dev = self.device
        ids = ids.to(device=dev, dtype=torch.int32).contiguous()
        labels = labels.to(device=dev, dtype=torch.int32).contiguous()
        boxes = boxes.to(device=dev, dtype=torch.float32).contiguous()
        counts = counts.to(device=dev, dtype=torch.int32).contiguous()
        sids = self._stream_ids(stream_ids, B, "Zones.update")
        E = int(max_events)
        inside = torch.empty(B, m, device=dev, dtype=torch.int32)
        occupancy = torch.empty(B, 32, device=dev, dtype=torch.int32)
        events = torch.empty(B, E, 5, device=dev, dtype=torch.int32)
        event_counts = torch.empty(B, device=dev, dtype=torch.int32)
        check(lib().lwdetr_zones_update(self._t, ptr(ids), ptr(labels), ptr(boxes), ptr(counts), B, m, ctypes.cast(sids, _vp), ptr(inside),
                                        ptr(occupancy), ptr(events) if E else None, E, ptr(event_counts), stream_ptr(dev)),
              "lwdetr_zones_update")
        return inside, occupancy, events, event_counts

    def export(self, stream):
        """Synchronous, waiting for this object's last update() or reset() and for nothing else on the device: one stream's
        state as a dict of numpy arrays: frame, overflow, line_counts int32 [L, num_classes + 1, 2] (in, out), entries int32
        [Z, num_classes + 1] (the last column: labels outside [0, num_classes)), and the records in ascending id: ids,
        last_seen, labels int32 [n], sides int8 [n, L], inside uint32 [n], entry int32 [n, Z] (entry frames, 0 outside)."""
        import numpy as np
        nc = int(self.params.num_classes) + 1
        cap = int(self.params.capacity)
        lc = np.zeros((32, nc, 2), np.int32)
        en = np.zeros((32, nc), np.int32)
        recs = (ZoneRecord * cap)()
        fo = (ctypes.c_int32 * 2)()
        info = (ctypes.c_int32 * 3)()
        check(lib().lwdetr_zones_export(self._t, int(stream), ctypes.cast(fo, _vp), ctypes.cast(info, _vp), lc.ctypes.data_as(_vp),
                                        en.ctypes.data_as(_vp), ctypes.cast(recs, _vp), cap), "lwdetr_zones_export")
        L, Z, n = list(info)
        raw = np.ctypeslib.as_array(recs)[:n]
        return dict(frame=fo[0], overflow=fo[1], line_counts=lc.reshape(-1)[:L * nc * 2].reshape(L, nc, 2).copy(),
                    entries=en.reshape(-1)[:Z * nc].reshape(Z, nc).copy(), ids=raw["id"].copy(), last_seen=raw["last_seen"].copy(),
                    labels=raw["label"].copy(), sides=raw["sides"][:, :L].copy(), inside=raw["inside"].copy(),
                    entry=raw["entry"][:, :Z].copy())


def homography(src, dst):
    """The 3x3 float64 homography H that maps four (x, y) frame pixels `src` to four ground points `dst` (metres, say):
    the 8x8 system of cv2.getPerspectiveTransform (h8 = 1) solved in float64, then H scaled by -1 if needed so that
    w = h6 x + h7 y + h8 > 0 at the centroid of src (lwdetr_speed's side of the horizon).  ValueError unless both are
    four finite points with no three of either collinear."""
    import numpy as np
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    for name, p in (("src", src), ("dst", dst)):
        if p.shape != (4, 2) or not np.isfinite(p).all():
            raise ValueError("homography: %s must be four finite (x, y) points, got shape %s" % (name, p.shape))
        for i in range(4):
            a, b, c = (p[k] for k in range(4) if k != i)
            if (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]) == 0:
                raise ValueError("homography: three points of %s are collinear" % name)
    A = np.zeros((8, 8))
    rhs = np.zeros(8)
    for i, ((x, y), (u, v)) in enumerate(zip(src, dst)):
        A[i] = (x, y, 1, 0, 0, 0, -x * u, -y * u)
        A[i + 4] = (0, 0, 0, x, y, 1, -x * v, -y * v)
        rhs[i], rhs[i + 4] = u, v
    try:
        H = np.append(np.linalg.solve(A, rhs), 1.0).reshape(3, 3)
    except np.linalg.LinAlgError:
        raise ValueError("homography: the points give a singular system") from None
    cx, cy = src.mean(0)
    if H[2, 0] * cx + H[2, 1] * cy + H[2, 2] < 0:
        H = -H
    return H


def _check_homography(H):
    """H as a contiguous float64 [3, 3] array, with lwdetr_speed_set's checks (finite, determinant neither 0 nor
    non-finite, in the header's order of operations); else ValueError."""
    import numpy as np
    h = np.ascontiguousarray(np.asarray(H, np.float64))
    if h.shape != (3, 3):
        raise ValueError("SpeedEstimator.set: the homography must be [3, 3], got %s" % (h.shape,))
    if not np.isfinite(h).all():
        raise ValueError("SpeedEstimator.set: the homography has a non-finite entry")
    f = [float(v) for v in h.reshape(-1)]
    det = f[0] * (f[4] * f[8] - f[5] * f[7]) - f[1] * (f[3] * f[8] - f[5] * f[6]) + f[2] * (f[3] * f[7] - f[4] * f[6])
    if det == 0.0 or not np.isfinite(det):
        raise ValueError("SpeedEstimator.set: the homography is singular")
    return h


class SpeedEstimator(_DeviceObject):
    """Ground-plane position, velocity and speed of each track per camera stream on the device (lwdetr_speed_*, the
    contract in include/lwdetr_b200.h, restated in tools/speed_spec.py): supervision's speed estimation, fed by
    Tracker.update.  capacity (records per stream, default 1024), window (samples per track, default 30), min_samples
    (default 15), forget_after (frames, default 30), anchor (an anchor index or a name of ANCHORS, default
    "bottom_center"), frame_rate (the clock of frames without timestamps, default 30).  Each stream's homography maps
    frame pixels to ground units (set(); default the identity: pixels per second).  All calls of one object must run on
    one CUDA stream (the current one at each call)."""

    RESET, DESTROY = "lwdetr_speed_reset", "lwdetr_speed_destroy"

    def __init__(self, num_streams, device=None, capacity=1024, window=30, min_samples=15, forget_after=30, anchor="bottom_center",
                 frame_rate=30.0):
        import torch
        if isinstance(anchor, str):
            anchor = ANCHORS.index(anchor)
        self.num_streams = int(num_streams)
        self.capacity, self.window = int(capacity), int(window)
        self.min_samples, self.forget_after, self.anchor = int(min_samples), int(forget_after), int(anchor)
        self.frame_rate = float(frame_rate)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._t = _vp()
        with torch.cuda.device(self.device):
            check(lib().lwdetr_speed_create(self.num_streams, self.capacity, self.window, self.min_samples, self.forget_after,
                                            self.anchor, self.frame_rate, ctypes.byref(self._t)), "lwdetr_speed_create")

    def set(self, stream, homography):
        """Replaces one stream's homography (a [3, 3] array, frame pixels -> ground units; checked before any device call).
        The history is kept.  Synchronous: waits for this object's last launch only.  Not during a stream capture."""
        stream = int(stream)
        if not 0 <= stream < self.num_streams:
            raise ValueError("SpeedEstimator.set: stream %d outside [0, %d)" % (stream, self.num_streams))
        h = _check_homography(homography)
        check(lib().lwdetr_speed_set(self._t, stream, h.ctypes.data_as(_vp)), "lwdetr_speed_set")

    def update(self, ids, boxes, counts, stream_ids=None, timestamps=None):
        """One frame for each of B distinct streams, on Tracker.update's outputs as they are: ids int32 [B, max_out], xyxy
        boxes fp32 [B, max_out, 4], counts [B] (CUDA; stream_ids default range(B)); timestamps: float64 [B] seconds (CUDA
        tensor, or a host sequence) or None (frame / frame_rate) -> (kin fp32 [B, max_out, 5] = (X, Y, vX, vY, speed),
        samples int32 [B, max_out]).  Stream-ordered, no synchronisation (a host timestamps sequence is copied to the
        device first); graph-safe with a CUDA tensor or None."""
        import torch
        B, m = ids.shape
        if tuple(boxes.shape) != (B, m, 4) or tuple(counts.shape) != (B,):
            raise RuntimeError("SpeedEstimator.update: ids %s, boxes %s and counts %s do not describe one [B, max_out] set"
                               % (tuple(ids.shape), tuple(boxes.shape), tuple(counts.shape)))
        dev = self.device
        ids = ids.to(device=dev, dtype=torch.int32).contiguous()
        boxes = boxes.to(device=dev, dtype=torch.float32).contiguous()
        counts = counts.to(device=dev, dtype=torch.int32).contiguous()
        if timestamps is not None:
            timestamps = torch.as_tensor(timestamps, dtype=torch.float64).to(dev).contiguous()
            if tuple(timestamps.shape) != (B,):
                raise RuntimeError("SpeedEstimator.update: timestamps must be [%d], got %s" % (B, tuple(timestamps.shape)))
        sids = self._stream_ids(stream_ids, B, "SpeedEstimator.update")
        kin = torch.empty(B, m, 5, device=dev, dtype=torch.float32)
        samples = torch.empty(B, m, device=dev, dtype=torch.int32)
        check(lib().lwdetr_speed_update(self._t, ptr(ids), ptr(boxes), ptr(counts), B, m, ctypes.cast(sids, _vp),
                                        ptr(timestamps) if timestamps is not None else None, ptr(kin), ptr(samples), stream_ptr(dev)),
              "lwdetr_speed_update")
        return kin, samples

    def export(self, stream):
        """Synchronous, waiting for this object's last update() or reset() and for nothing else on the device: one stream's
        state as a dict: frame, records, overflow, clock_errors, last_t, homography float64 [3, 3], and the records in
        ascending id: ids, last_seen int32 [n], and samples, a list of float64 [n_i, 3] arrays (t, x, y), oldest first."""
        import numpy as np
        cap, W = self.capacity, self.window
        head = (ctypes.c_int32 * 4)()
        last_t = ctypes.c_double()
        H = np.zeros(9, np.float64)
        ids = np.zeros(cap, np.int32)
        seen = np.zeros(cap, np.int32)
        counts = np.zeros(cap, np.int32)
        samples = np.zeros((cap, W, 3), np.float64)
        check(lib().lwdetr_speed_export(self._t, int(stream), ctypes.cast(head, _vp), ctypes.byref(last_t), H.ctypes.data_as(_vp),
                                        ids.ctypes.data_as(_vp), seen.ctypes.data_as(_vp), counts.ctypes.data_as(_vp),
                                        samples.ctypes.data_as(_vp), cap), "lwdetr_speed_export")
        n = head[1]
        return dict(frame=head[0], records=n, overflow=head[2], clock_errors=head[3], last_t=last_t.value, homography=H.reshape(3, 3),
                    ids=ids[:n].copy(), last_seen=seen[:n].copy(), samples=[samples[i, :counts[i]].copy() for i in range(n)])


LABEL_NAME, LABEL_ID, LABEL_SCORE = 1, 2, 4
ANNOTATOR_OPTIONS = ("thickness", "text_scale", "box_fill_alpha", "label", "zone_fill_alpha", "zone_thickness", "privacy_block")


class Annotator(_DeviceObject):
    """Draws detections, tracks and zones into RGB or NV12 frames in place on the device, with privacy pixelation
    (lwdetr_annotator_* / lwdetr_annotate, the contract in include/lwdetr_b200.h, restated in tools/annotate_spec.py).
    names: class names (list, at most 31 ASCII characters each; default the class id); palette: RGB triples (1 to 256;
    default the header's 16); privacy: labels whose boxes are pixelated instead of drawn; options: thickness, text_scale,
    box_fill_alpha, label (a mask of LABEL_*), zone_fill_alpha, zone_thickness, privacy_block.  All calls of one object must
    run on one CUDA stream (the current one at each call)."""

    DESTROY = "lwdetr_annotator_destroy"

    def __init__(self, num_classes, names=None, palette=None, privacy=(), device=None, **options):
        import torch
        bad = set(options) - set(ANNOTATOR_OPTIONS)
        if bad:
            raise RuntimeError("Annotator: unknown options %s" % ", ".join(sorted(bad)))
        self.num_classes = int(num_classes)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._t = _vp()
        with torch.cuda.device(self.device):
            check(lib().lwdetr_annotator_create(self.num_classes, ctypes.byref(self._t)), "lwdetr_annotator_create")
        for n, v in options.items():
            self.set_option(n, v)
        if names is not None:
            self.set_names(names)
        if palette is not None:
            self.set_palette(palette)
        if privacy:
            self.set_privacy(privacy)

    def set_option(self, name, value):
        check(lib().lwdetr_annotator_set_option(self._t, name.encode(), int(value)), "lwdetr_annotator_set_option")

    def set_names(self, names):
        """Synchronous (waits for this object's last draw only)."""
        names = list(names)
        if any("\n" in n for n in names):
            raise RuntimeError("Annotator.set_names: a name cannot hold a newline")
        check(lib().lwdetr_annotator_set_names(self._t, "\n".join(names).encode("ascii", "replace")), "lwdetr_annotator_set_names")

    def set_palette(self, palette):
        import numpy as np
        arr = np.ascontiguousarray(np.asarray(palette, np.uint8).reshape(-1, 3))
        check(lib().lwdetr_annotator_set_palette(self._t, arr.ctypes.data_as(_vp), len(arr)), "lwdetr_annotator_set_palette")

    def set_privacy(self, classes):
        arr, n = self._ids(classes)
        check(lib().lwdetr_annotator_set_privacy(self._t, ctypes.cast(arr, _vp), n), "lwdetr_annotator_set_privacy")

    def annotate(self, frames, scores, labels, boxes, ids=None, counts=None, streams=None, zones=None, occupancy=None,
                 score_threshold=0.0, colorspace=None):
        """lwdetr_annotate(_nv12) on device arrays as they are: scores fp32 [B, k], labels int32 [B, k], boxes fp32 [B, k, 4],
        ids int32 [B, k] or None, counts int32 [B] or None, occupancy int32 [B, 32] or None (Zones.update's), all CUDA; the
        frames (RGB or NV12 as capi.Frames takes them, CUDA, never copied) are drawn in place.  streams: the frames' stream
        ids in zones (default range(B)).  Stream-ordered, no synchronisation; graph-safe."""
        import torch
        fb = frames if isinstance(frames, Frames) else Frames(frames, self.device, colorspace)
        if fb.device != self.device:
            raise RuntimeError("Annotator: frames on %s, the annotator on %s" % (fb.device, self.device))
        B = len(fb.items)
        if scores.dim() != 2 or scores.shape[0] != B:
            raise RuntimeError("Annotator: scores must be [%d, k], got %s" % (B, tuple(scores.shape)))
        k = scores.shape[1]
        shapes = [(labels, (B, k)), (boxes, (B, k, 4))] + [(t, sh) for t, sh in ((ids, (B, k)), (counts, (B,)), (occupancy, (B, 32)))
                                                           if t is not None]
        for t, sh in shapes:
            if tuple(t.shape) != sh:
                raise RuntimeError("Annotator: expected %s, got %s" % (sh, tuple(t.shape)))
        args = [t if t is None else t.to(device=self.device, dtype=dt).contiguous()
                for t, dt in ((ids, torch.int32), (scores, torch.float32), (labels, torch.int32), (boxes, torch.float32),
                              (counts, torch.int32), (occupancy, torch.int32))]
        sids = None
        if zones is not None:
            arr, n = self._ids(range(B) if streams is None else streams)
            if n != B:
                raise RuntimeError("Annotator: %d stream ids for %d frames" % (n, B))
            sids = ctypes.cast(arr, _vp)
        name = "lwdetr_annotate_nv12" if fb.nv12 else "lwdetr_annotate"
        ids_, sc, lab, bx, cn, occ = args
        check(getattr(lib(), name)(self._t, fb.descs(fb.sizes), B, ptr(ids_), ptr(sc), ptr(lab), ptr(bx), ptr(cn), k,
                                   float(score_threshold), zones._t if zones is not None else None, sids, ptr(occ),
                                   stream_ptr(self.device)), name)

    def draw(self, frames, dets, streams=None, zones=None, score_threshold=0.0, colorspace=None):
        """Draws detect() / detect_tiled() / track()'s per-frame lists into the frames in place: each dict's "scores",
        "labels", "boxes" and, when present, "ids" (colour by track id and "#id" in the label; otherwise colour by class)
        and "occupancy" (with zones).  The lists are packed on the device; nothing is read back."""
        import torch
        fb = frames if isinstance(frames, Frames) else Frames(frames, self.device, colorspace)
        B = len(fb.items)
        if len(dets) != B:
            raise RuntimeError("Annotator.draw: %d detection lists for %d frames" % (len(dets), B))
        dev = self.device
        n = [int(d["scores"].shape[0]) for d in dets]
        k = max(max(n), 1)
        if k > 1024:
            raise RuntimeError("Annotator.draw: at most 1024 entries per frame, got %d" % k)
        with_ids = all("ids" in d for d in dets)
        scores = torch.zeros(B, k, device=dev, dtype=torch.float32)
        labels = torch.zeros(B, k, device=dev, dtype=torch.int32)
        boxes = torch.zeros(B, k, 4, device=dev, dtype=torch.float32)
        ids = torch.zeros(B, k, device=dev, dtype=torch.int32) if with_ids else None
        for b, d in enumerate(dets):
            c = n[b]
            scores[b, :c] = d["scores"]
            labels[b, :c] = d["labels"].to(torch.int32)
            boxes[b, :c] = d["boxes"].reshape(-1, 4)
            if with_ids:
                ids[b, :c] = d["ids"].to(torch.int32)
        counts = torch.tensor(n, dtype=torch.int32).to(dev)
        occ = None
        if zones is not None and all("occupancy" in d for d in dets):
            occ = torch.stack([d["occupancy"].to(device=dev, dtype=torch.int32) for d in dets])
        self.annotate(fb, scores, labels, boxes, ids=ids, counts=counts, streams=streams, zones=zones, occupancy=occ,
                      score_threshold=score_threshold)


def layernorm_e4m3(x, eps=1e-6):
    """x: CUDA fp16 [rows, C] (any row stride) -> (e4m3 codes uint8 [rows, C], fp32 row scales [rows]); see
    lwdetr_layernorm_e4m3."""
    import torch
    if x.dtype != torch.float16:
        raise RuntimeError("layernorm_e4m3: x must be float16, got %s" % x.dtype)
    rows, C = x.shape
    q = torch.empty(rows, C, device=x.device, dtype=torch.uint8)
    s = torch.empty(rows, device=x.device, dtype=torch.float32)
    check(lib().lwdetr_layernorm_e4m3(ptr(x), x.stride(0), rows, C, float(eps), ptr(q), q.stride(0), ptr(s), stream_ptr(x.device)),
          "lwdetr_layernorm_e4m3")
    return q, s


def gemm_e4m3(A, a_scale, W, w_scale, bias=None, act=ACT_NONE, out=None):
    """out fp16 [M, N] = act(a_scale[m] * w_scale[n] * (A @ W.T) + bias); A uint8 e4m3 codes [M, K] (row stride a multiple of
    16), W uint8 [N, K] contiguous, scales / bias fp32 (lwdetr_gemm_e4m3)."""
    import torch
    M, K = A.shape
    N = W.shape[0]
    if out is None:
        out = torch.empty(M, N, device=A.device, dtype=torch.float16)
    check(lib().lwdetr_gemm_e4m3(ptr(A), A.stride(0), ptr(a_scale), M, K, ptr(W), ptr(w_scale), N, ptr(bias), act, ptr(out),
                                 out.stride(0), stream_ptr(A.device)), "lwdetr_gemm_e4m3")
    return out


def vit_mlp(x, stats_in, W1, colsum1, b1, W2, b2=None, gamma=None, eps=1e-6, out=None, stats_out=None):
    """Fused ViT MLP of the 192-wide encoder (lwdetr_vit_mlp): out = x + gamma * (round16(gelu(LN-fold(x W1^T) + b1)) W2^T + b2).
    x 16-bit [M, 192] (row stride a multiple of 16), stats_in fp32 [M, parts, 2] LayerNorm partials, W1 [768, 192] and W2
    [192, 768] contiguous in x's dtype, colsum1 / b1 / b2 / gamma fp32; out [M, 192] (any row stride that is a multiple of
    16) and stats_out fp32 [M, 2 or 6, 2] optional."""
    import torch
    M = x.shape[0]
    if out is None:
        out = torch.empty(M, 192, device=x.device, dtype=x.dtype)
    parts_out = 0 if stats_out is None else stats_out.shape[1]
    check(lib().lwdetr_vit_mlp(kernel_dtype_code(x.dtype), ptr(x), x.stride(0), M, ptr(stats_in), stats_in.shape[1], float(eps),
                               ptr(W1), ptr(colsum1), ptr(b1), ptr(W2), ptr(b2), ptr(gamma), ptr(out), out.stride(0),
                               ptr(stats_out), parts_out, stream_ptr(x.device)), "lwdetr_vit_mlp")
    return out


def host_quant_e4m3_rows(src):
    """src: CPU fp32 [rows, K] -> (e4m3 codes uint8 [rows, K], fp32 scales [rows]), the weight quantiser of the e4m3 mode."""
    import torch
    src = src.detach().to("cpu", torch.float32).contiguous()
    rows, K = src.shape
    q = torch.empty(rows, K, dtype=torch.uint8)
    s = torch.empty(rows, dtype=torch.float32)
    check(lib().lwdetr_host_quant_e4m3_rows(ptr(src), rows, K, ptr(q), ptr(s)), "lwdetr_host_quant_e4m3_rows")
    return q, s


def host_bicubic(src, n_out):
    """src: CPU fp32 [n, n, C] -> [n_out, n_out, C] (no GPU involved)."""
    import torch
    src = src.contiguous().float()
    dst = torch.empty(n_out, n_out, src.shape[2], dtype=torch.float32)
    check(lib().lwdetr_host_bicubic(ptr(src), src.shape[0], src.shape[2], n_out, ptr(dst)), "lwdetr_host_bicubic")
    return dst


def host_bicubic_hw(src, out_h, out_w):
    """src: CPU fp32 [n, n, C] -> [out_h, out_w, C] (no GPU involved)."""
    import torch
    src = src.contiguous().float()
    dst = torch.empty(out_h, out_w, src.shape[2], dtype=torch.float32)
    check(lib().lwdetr_host_bicubic_hw(ptr(src), src.shape[0], src.shape[2], out_h, out_w, ptr(dst)), "lwdetr_host_bicubic_hw")
    return dst


ConfigStruct = _STRUCTS["lwdetr_config"]


InputDesc = _STRUCTS["lwdetr_input"]


IN_F32_NCHW, IN_16_NCHW, IN_U8_NHWC = 0, 1, 2
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)      # demo/demo.py:150-153, datasets/coco.py


FrameStruct = _STRUCTS["lwdetr_frame"]


def frame_list(frames, device=None):
    """Raw frames as a list of CUDA uint8 [h, w, 3] tensors: takes that list or one [B, h, w, 3] tensor.  A frame may be a
    view (a crop of a larger surface) as long as its pixels are packed RGB: stride(2) == 1 and stride(1) == 3."""
    import torch
    if isinstance(frames, torch.Tensor):
        if frames.dim() != 4:
            raise RuntimeError("lwdetr_b200: a frame batch must be [B, h, w, 3], got %s" % (tuple(frames.shape),))
        frames = list(frames.unbind(0))
    frames = list(frames)
    if not frames:
        raise RuntimeError("lwdetr_b200: no frames")
    for i, f in enumerate(frames):
        if not isinstance(f, torch.Tensor) or f.dtype != torch.uint8:
            raise RuntimeError("lwdetr_b200: frame %d must be a uint8 tensor, got %s" % (i, getattr(f, "dtype", type(f))))
        if f.dim() != 3 or f.shape[2] != 3:
            raise RuntimeError("lwdetr_b200: frame %d must be [h, w, 3] (HWC), got %s" % (i, tuple(f.shape)))
        if f.device.type != "cuda" or (device is not None and f.device != device):
            raise RuntimeError("lwdetr_b200: frame %d is on %s; frames must be CUDA tensors%s"
                               % (i, f.device, "" if device is None else " on %s" % (device,)))
        if f.stride(2) != 1 or f.stride(1) != 3 or f.stride(0) < 3 * f.shape[1]:
            raise RuntimeError("lwdetr_b200: frame %d has strides %s; packed RGB pixels are required: stride(2) == 1, "
                               "stride(1) == 3, stride(0) >= 3 * width" % (i, tuple(f.stride())))
    return frames


def frame_descs(frames, dsts):
    """HOST array of lwdetr_frame for frame_list() tensors and their (dst_h, dst_w)."""
    arr = (FrameStruct * len(frames))()
    for d, f, (dh, dw) in zip(arr, frames, dsts):
        d.data, d.height, d.width, d.pitch_bytes, d.dst_h, d.dst_w = f.data_ptr(), f.shape[0], f.shape[1], f.stride(0), int(dh), int(dw)
    return arr


FrameNV12Struct = _STRUCTS["lwdetr_frame_nv12"]


# colorspace names of NV12 frames -> LWDETR_CSC_* (include/lwdetr_b200.h): limited (studio) range unless "_full"
COLORSPACES = {"bt601": 0, "bt709": 1, "bt601_full": 2, "bt709_full": 3}


def _is_nv12(f):
    import torch
    return isinstance(f, (tuple, list)) or (isinstance(f, torch.Tensor) and f.dim() == 2)


def _check_plane(i, name, t, rows, row_bytes, device):
    import torch
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 2:
        raise RuntimeError("lwdetr_b200: NV12 frame %d: %s must be a 2-D uint8 tensor, got %s" % (i, name, getattr(t, "dtype", type(t))))
    if tuple(t.shape) != (rows, row_bytes):
        raise RuntimeError("lwdetr_b200: NV12 frame %d: %s must be [%d, %d], got %s" % (i, name, rows, row_bytes, tuple(t.shape)))
    if t.stride(1) != 1 or (rows > 1 and t.stride(0) < row_bytes):
        raise RuntimeError("lwdetr_b200: NV12 frame %d: %s has strides %s; stride(1) == 1 and stride(0) >= %d are required"
                           % (i, name, tuple(t.stride()), row_bytes))
    if t.device.type != "cuda" or (device is not None and t.device != device):
        raise RuntimeError("lwdetr_b200: NV12 frame %d: %s is on %s; frames must be CUDA tensors%s"
                           % (i, name, t.device, "" if device is None else " on %s" % (device,)))


def nv12_list(frames, device=None):
    """NV12 frames as a list of (luma [h, w], chroma [ceil(h/2), 2 * ceil(w/2)]) CUDA uint8 pairs (each plane any row stride,
    stride(1) == 1).  Takes that list, packed NV12 frames [3h/2, w] (h and w even; split into their two planes here) in the
    list, or one packed [B, 3h/2, w] tensor."""
    import torch
    if isinstance(frames, torch.Tensor):
        frames = list(frames.unbind(0))
    pairs = []
    for i, f in enumerate(frames):
        if isinstance(f, torch.Tensor):
            rows, w = f.shape
            h = rows * 2 // 3
            if rows % 3 or h % 2 or w % 2:
                raise RuntimeError("lwdetr_b200: packed NV12 frame %d is %s; [3h/2, w] with h and w even is required (odd sizes: pass "
                                   "the (luma, chroma) planes)" % (i, tuple(f.shape)))
            f = (f[:h], f[h:])
        if len(f) != 2:
            raise RuntimeError("lwdetr_b200: NV12 frame %d must be a (luma, chroma) pair" % i)
        luma, chroma = f
        if not isinstance(luma, torch.Tensor) or luma.dim() != 2:
            raise RuntimeError("lwdetr_b200: NV12 frame %d: luma must be a 2-D uint8 tensor [h, w]" % i)
        h, w = luma.shape
        _check_plane(i, "luma", luma, h, w, device)
        _check_plane(i, "chroma", chroma, (h + 1) // 2, 2 * ((w + 1) // 2), luma.device)
        pairs.append((luma, chroma))
    return pairs


def colorspace_codes(colorspace, B):
    """LWDETR_CSC_* code of each of B NV12 frames from one name or one name per frame."""
    if colorspace is None:
        raise RuntimeError("lwdetr_b200: NV12 frames need colorspace= (one of %s, or one per frame): there is no safe default, a "
                           "wrong matrix shifts every colour" % ", ".join(COLORSPACES))
    names = [colorspace] * B if isinstance(colorspace, str) else list(colorspace)
    if len(names) != B:
        raise RuntimeError("lwdetr_b200: %d colorspaces for %d frames" % (len(names), B))
    for n in names:
        if n not in COLORSPACES:
            raise RuntimeError("lwdetr_b200: unknown colorspace %r; one of %s" % (n, ", ".join(COLORSPACES)))
    return [COLORSPACES[n] for n in names]


class Frames:
    """One batch of raw frames, RGB (frame_list) or NV12 (nv12_list), told apart by their form.  colorspace is required for
    NV12 frames and rejected for RGB ones.  .sizes: each frame's (h, w); .descs(dsts): the HOST descriptor array of the C ABI."""

    def __init__(self, frames, device=None, colorspace=None):
        import torch
        if isinstance(frames, Frames):
            self.__dict__.update(frames.__dict__)
            return
        if isinstance(frames, torch.Tensor):
            self.nv12 = frames.dim() == 3 and frames.shape[2] != 3      # [B, 3h/2, w]; [h, w, 3] is an RGB frame without its batch axis
        else:
            frames = list(frames)
            kinds = {_is_nv12(f) for f in frames}
            if len(kinds) > 1:
                raise RuntimeError("lwdetr_b200: one call takes RGB or NV12 frames, not a mix of both")
            self.nv12 = kinds == {True}
        if self.nv12:
            self.codes = colorspace_codes(colorspace, len(frames))
            self.items = nv12_list(frames, device)
            self.sizes = [(y.shape[0], y.shape[1]) for y, _ in self.items]
        else:
            if colorspace is not None:
                raise RuntimeError("lwdetr_b200: colorspace applies to NV12 frames only; these frames are RGB")
            self.items = frame_list(frames, device)
            self.sizes = [(f.shape[0], f.shape[1]) for f in self.items]
        self.device = self.items[0][0].device if self.nv12 else self.items[0].device

    def select(self, rows):
        """The frames at positions `rows`, as one Frames (nothing copied)."""
        out = Frames.__new__(Frames)
        out.__dict__.update(self.__dict__)
        out.items = [self.items[i] for i in rows]
        out.sizes = [self.sizes[i] for i in rows]
        if self.nv12:
            out.codes = [self.codes[i] for i in rows]
        return out

    def descs(self, dsts):
        """ctypes pointer to the HOST array of lwdetr_frame / lwdetr_frame_nv12 for these frames and their (dst_h, dst_w)."""
        if not self.nv12:
            return ctypes.cast(frame_descs(self.items, dsts), _vp)
        arr = (FrameNV12Struct * len(self.items))()
        self._arr = arr
        for d, (y, c), cs, (dh, dw) in zip(arr, self.items, self.codes, dsts):
            d.luma, d.luma_pitch, d.chroma, d.chroma_pitch = y.data_ptr(), y.stride(0), c.data_ptr(), c.stride(0)
            d.height, d.width, d.dst_h, d.dst_w, d.colorspace = y.shape[0], y.shape[1], int(dh), int(dw), cs
        return ctypes.cast(arr, _vp)


def _norm3(v):
    return (ctypes.c_float * 3)(*[float(x) for x in v])


def resize_patches(frames, dsts, size, dtype, mean=None, std=None, want_mask=False, colorspace=None):
    """lwdetr_resize_patches(_nv12): frames (RGB or NV12, see Frames) resized to their dsts on an (H, W) = size canvas ->
    (window-major patch matrix [B*(H/16)*(W/16), 768] in `dtype`, padding mask bool [B, H, W] or None)."""
    import torch
    fb = Frames(frames, colorspace=colorspace)
    H, W = int(size[0]), int(size[1])
    dev, B = fb.device, len(fb.items)
    mean, std = IMAGENET_MEAN if mean is None else mean, IMAGENET_STD if std is None else std
    A = torch.empty(max(B * (H // 16) * (W // 16), 1), 768, device=dev, dtype=dtype)
    mask = torch.empty(B, H, W, device=dev, dtype=torch.bool) if want_mask else None
    name = "lwdetr_resize_patches_nv12" if fb.nv12 else "lwdetr_resize_patches"
    check(getattr(lib(), name)(kernel_dtype_code(dtype), fb.descs(dsts), B, H, W, ctypes.cast(_norm3(mean), _vp),
                               ctypes.cast(_norm3(std), _vp), ptr(A), ptr(mask), stream_ptr(dev)), name)
    return A, mask


CROP_FILTERS = {"bilinear": 0, "antialias": 1}     # LWDETR_CROP_BILINEAR (cv2 INTER_LINEAR) / LWDETR_CROP_ANTIALIAS (PIL triangle)


def crops(frames, boxes, frame_index, size=(256, 128), filter="bilinear", mean=None, std=None, normalize=True, dtype=None,
          count=None, colorspace=None, out=None, valid=None):
    """lwdetr_crops(_nv12): each box cut out of its frame on the device and resized to size = (h, w) (include/lwdetr_b200.h).
    frames: RGB or NV12 (capi.Frames, or frames as Frames takes them with colorspace); boxes fp32 [N, 4] xyxy in frame pixels
    and frame_index int [N] (CUDA).  filter "bilinear" (cv2.resize INTER_LINEAR, BoT-SORT / FastReID) or "antialias" (the PIL
    triangle filter of the frame path, any downscale).  normalize: (v / 255 - mean) / std (default ImageNet's), else the
    level 0..255 itself.  dtype float32 (default), float16 or bfloat16.  count: CUDA int32 [1]; crops at or past it are not
    written (out / valid may be passed to keep their earlier contents there).  Returns (crops [N, 3, h, w], valid bool [N]):
    an invalid crop (empty or non-finite box) is zeros.  Stream-ordered, no synchronisation."""
    import torch
    if filter not in CROP_FILTERS:
        raise RuntimeError("crops: filter must be one of %s, got %r" % (", ".join(CROP_FILTERS), filter))
    fb = frames if isinstance(frames, Frames) else Frames(frames, colorspace=colorspace)
    dev, B = fb.device, len(fb.items)
    dtype = torch.float32 if dtype is None else dtype
    code = _et_code(dtype, "crops: dtype")
    if boxes.dim() != 2 or boxes.shape[1] != 4 or tuple(frame_index.shape) != (boxes.shape[0],):
        raise RuntimeError("crops: boxes must be [N, 4] and frame_index [N], got %s and %s" % (tuple(boxes.shape), tuple(frame_index.shape)))
    N = boxes.shape[0]
    h, w = int(size[0]), int(size[1])
    boxes = boxes.to(device=dev, dtype=torch.float32).contiguous()
    fidx = frame_index.to(device=dev, dtype=torch.int32).contiguous()
    if out is None:
        out = torch.empty(N, 3, h, w, device=dev, dtype=dtype)
    if valid is None:
        valid = torch.empty(N, device=dev, dtype=torch.int8)
    if tuple(out.shape) != (N, 3, h, w) or out.dtype != dtype or not out.is_contiguous() or valid.dtype != torch.int8 or valid.numel() != N:
        raise RuntimeError("crops: out must be a contiguous [%d, 3, %d, %d] %s tensor and valid int8 [%d]" % (N, h, w, dtype, N))
    if count is not None:
        count = count.to(device=dev, dtype=torch.int32).contiguous()
    mean, std = IMAGENET_MEAN if mean is None else mean, IMAGENET_STD if std is None else std
    if N:
        name = "lwdetr_crops_nv12" if fb.nv12 else "lwdetr_crops"
        check(getattr(lib(), name)(fb.descs(fb.sizes), B, ptr(boxes), ptr(fidx), N, ptr(count), h, w, CROP_FILTERS[filter],
                                   1 if normalize else 0, ctypes.cast(_norm3(mean), _vp), ctypes.cast(_norm3(std), _vp), code, ptr(out),
                                   ptr(valid), stream_ptr(dev)), name)
    return out, valid.view(torch.bool)


def crop_select(scores, boxes, sizes, threshold):
    """lwdetr_crop_select: the entries (scores fp32 [B, k], xyxy boxes fp32 [B, k, 4], CUDA; sizes: each frame's (h, w)) with
    score > threshold and a valid crop, in (frame, entry) order -> (frame int32 [B*k], entry int32 [B*k] (flat b * k + j),
    boxes fp32 [B*k, 4], count int32 [1]), all CUDA; rows at or past the count are not written.  No synchronisation."""
    import torch
    B, k = scores.shape
    if tuple(boxes.shape) != (B, k, 4) or len(sizes) != B:
        raise RuntimeError("crop_select: scores %s, boxes %s and %d frame sizes do not describe one [B, k] set"
                           % (tuple(scores.shape), tuple(boxes.shape), len(sizes)))
    dev = scores.device
    scores = scores.to(dtype=torch.float32).contiguous()
    boxes = boxes.to(device=dev, dtype=torch.float32).contiguous()
    hw = (ctypes.c_int32 * (2 * B))(*[int(v) for s in sizes for v in s])
    frame = torch.empty(B * k, device=dev, dtype=torch.int32)
    entry = torch.empty(B * k, device=dev, dtype=torch.int32)
    sel = torch.empty(B * k, 4, device=dev, dtype=torch.float32)
    count = torch.empty(1, device=dev, dtype=torch.int32)
    check(lib().lwdetr_crop_select(ptr(scores), ptr(boxes), B, k, ctypes.cast(hw, _vp), float(threshold), ptr(frame), ptr(entry), ptr(sel),
                                   ptr(count), stream_ptr(dev)), "lwdetr_crop_select")
    return frame, entry, sel, count


def scatter_rows(rows, entry, num_out, count=None):
    """lwdetr_scatter_rows: rows [N, D] (CUDA float32 / float16 / bfloat16, last dimension contiguous) -> [num_out, D] of
    the same dtype with row i (i < count, default N) at entry[i] and zeros elsewhere.  No synchronisation."""
    import torch
    N, D = rows.shape
    if rows.stride(1) != 1:
        rows = rows.contiguous()
    code = _et_code(rows.dtype, "scatter_rows: dtype")
    entry = entry.to(device=rows.device, dtype=torch.int32).contiguous()
    if entry.numel() < N:
        raise RuntimeError("scatter_rows: %d entries for %d rows" % (entry.numel(), N))
    out = torch.empty(int(num_out), D, device=rows.device, dtype=rows.dtype)
    if count is not None:
        count = count.to(device=rows.device, dtype=torch.int32).contiguous()
    if N == 0:
        return out.zero_()
    check(lib().lwdetr_scatter_rows(code, ptr(rows), rows.stride(0), D, ptr(entry), ptr(count), N, ptr(out), int(num_out),
                                    stream_ptr(rows.device)), "lwdetr_scatter_rows")
    return out


AuxOut = _STRUCTS["lwdetr_aux_out"]


def config_struct(cfg):
    c = ConfigStruct()
    c.vit_dim, c.vit_depth, c.vit_heads = cfg.vit_dim, cfg.vit_depth, cfg.vit_heads
    c.window_block_mask = sum(1 << i for i in cfg.window_blocks)
    taps = list(cfg.taps)
    c.n_taps = len(taps)
    for i, t in enumerate(taps):
        c.taps[i] = t
    c.n_levels = cfg.n_levels
    for i, p in enumerate(cfg.projector_scale):
        c.level_scale_log2[i] = {"P3": 1, "P4": 0, "P5": -1}[p]
    c.hidden_dim, c.sa_heads, c.ca_heads = cfg.hidden_dim, cfg.sa_nheads, cfg.ca_nheads
    c.dec_points, c.num_queries, c.dec_layers = cfg.dec_n_points, cfg.num_queries, cfg.dec_layers
    c.dim_feedforward, c.num_classes, c.group_detr, c.img_size = cfg.dim_feedforward, cfg.num_classes, cfg.group_detr, cfg.img_size
    return c


def check_topk_override(ov, B, nq, S, device):
    """The forced two-stage selection of one forward, checked: an integer tensor [B, nq] on the host or on the engine's
    `device` (not on any other device) whose every index lies in [0, S), S the memory length of the input size.  The engine
    gathers the encoder rows, class logits and proposals at these indices without a check of its own.  Returns it as
    contiguous int32 on `device` (a host tensor is copied there); RuntimeError naming the limit otherwise.  Costs one
    read-back of the minimum and maximum."""
    import torch
    if tuple(ov.shape) != (B, nq):
        raise RuntimeError("lwdetr_b200: topk_override must be [B, num_queries] = [%d, %d], got %s" % (B, nq, tuple(ov.shape)))
    if ov.dtype.is_floating_point or ov.dtype.is_complex or ov.dtype == torch.bool:
        raise RuntimeError("lwdetr_b200: topk_override must be an integer tensor, got %s" % (ov.dtype,))
    device = torch.device(device)
    if ov.device != device and ov.device.type != "cpu":
        raise RuntimeError("lwdetr_b200: topk_override is on %s but the engine lives on %s (pass it there or on the host)"
                           % (ov.device, device))
    lo, hi = torch.stack(torch.aminmax(ov.reshape(-1).long())).tolist()
    if lo < 0 or hi >= S:
        raise RuntimeError("lwdetr_b200: topk_override indices must lie in [0, %d) (the memory length of this input size), got "
                           "[%d, %d]" % (S, lo, hi))
    return ov.to(device=device, dtype=torch.int32).contiguous()


class Engine:
    """Owns one lwdetr_handle: packed weights + kernel schedule on the current CUDA device."""

    def __init__(self, cfg, dtype, device=None):
        """dtype: torch.float16, torch.bfloat16, or torch.float8_e4m3fn for the fp16 engine with the encoder's qkv / fc1 in
        e4m3 (outputs are the same fp32 dict in every mode)."""
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("lwdetr_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.cfg, self.dtype = cfg, dtype
        self._h = _vp()
        cs = config_struct(cfg)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        with torch.cuda.device(self.device):      # the handle binds to the device current at creation
            check(lib().lwdetr_create(ctypes.byref(cs), dtype_code(dtype), ctypes.byref(self._h)), "lwdetr_create")
        self._captures = []

    def close(self):
        if self._h:
            lib().lwdetr_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state_dict(self, sd):
        """sd: name -> tensor with the reference state_dict names (any device/dtype; copied to CPU fp32)."""
        import torch
        names, keep = [], []
        for k, v in sd.items():
            if not torch.is_floating_point(v):
                continue                                    # num_batches_tracked
            names.append(k.encode())
            keep.append(v.detach().to("cpu", torch.float32).contiguous())
        n = len(names)
        c_names = (ctypes.c_char_p * n)(*names)
        c_ptrs = (_vp * n)(*[t.data_ptr() for t in keep])
        c_numel = (ctypes.c_int64 * n)(*[t.numel() for t in keep])
        check(lib().lwdetr_load_weights(self._h, n, ctypes.cast(c_names, _vp), ctypes.cast(c_ptrs, _vp),
                                        ctypes.cast(c_numel, _vp)), "lwdetr_load_weights")

    def broadcast_weights(self, nccl_comm, root=0):
        """One ncclBroadcast of the packed arena from rank `root` (nccl_comm: integer ncclComm_t, see b200/dist.py)."""
        check(lib().lwdetr_broadcast_weights(self._h, ctypes.c_void_p(nccl_comm), int(root), stream_ptr()), "lwdetr_broadcast_weights")

    def arena_bytes(self):
        return int(lib().lwdetr_weight_arena_bytes(self._h))

    def set_option(self, name, value):
        check(lib().lwdetr_set_option(self._h, name.encode(), int(value)), "lwdetr_set_option")

    def forward(self, images, want_aux=True, topk_override=None, mask=None, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        """images: CUDA [B,3,H,W] fp32 / compute dtype, or CUDA uint8 [B,H,W,3] (HWC, normalised on the fly with mean/std);
        mask: CUDA bool [B,H,W] (True = padded pixel) or None.  H and W: multiples of 64 in [128, 1344] (b200.config.
        check_input_size); a size other than the previous call's re-plans the engine.  Returns the reference's output dict
        (fp32 CUDA tensors)."""
        import torch
        from .config import check_input_size
        if images.device.type != "cuda":
            raise RuntimeError("lwdetr_b200: images must be CUDA tensors")
        if images.device != self.device:
            raise RuntimeError("lwdetr_b200: images are on %s but the engine lives on %s" % (images.device, self.device))
        desc = InputDesc()
        if images.dtype == torch.uint8:
            if images.dim() != 4 or images.shape[3] != 3:
                raise RuntimeError("lwdetr_b200: uint8 images must be [B, H, W, 3] (HWC), got %s" % (tuple(images.shape),))
            H, W = int(images.shape[1]), int(images.shape[2])
            desc.format = IN_U8_NHWC
            for c in range(3):
                desc.mean[c], desc.std[c] = float(mean[c]), float(std[c])
        else:
            if images.dim() != 4 or images.shape[1] != 3:
                raise RuntimeError("lwdetr_b200: expected images [B, 3, H, W], got %s" % (tuple(images.shape),))
            H, W = int(images.shape[2]), int(images.shape[3])
            if images.dtype not in (torch.float32, io_dtype(self.dtype)):
                images = images.float()
            desc.format = IN_F32_NCHW if images.dtype == torch.float32 else IN_16_NCHW
        check_input_size(self.cfg, H, W)
        images = images.contiguous()
        mk = None
        if mask is not None:
            if tuple(mask.shape) != (images.shape[0], H, W):
                raise RuntimeError("lwdetr_b200: mask must be [B, %d, %d], got %s" % (H, W, tuple(mask.shape)))
            mk = mask.to(device=self.device, dtype=torch.bool).contiguous()
        desc.images = images.data_ptr()
        desc.padding_mask = mk.data_ptr() if mk is not None else None
        B, dev = images.shape[0], images.device
        res, logits, boxes, aux = self._outputs(B, dev, want_aux)
        ov = None
        if topk_override is not None:
            ov = check_topk_override(topk_override, B, self.cfg.num_queries, self.cfg.memory_len_at(H, W), self.device)
        check(lib().lwdetr_forward_hw(self._h, ctypes.byref(desc), B, H, W, ptr(logits), ptr(boxes),
                                      ctypes.byref(aux) if aux is not None else None, ptr(ov), stream_ptr(self.device)), "lwdetr_forward_hw")
        self._last_inputs = (images, ov, mk)    # keep alive until the stream has consumed them
        return res

    def _outputs(self, B, dev, want_aux):
        """Output tensors of one forward: (result dict, pred_logits, pred_boxes, AuxOut or None)."""
        import torch
        nq, nc, nl = self.cfg.num_queries, self.cfg.num_classes, self.cfg.dec_layers
        logits = torch.empty(B, nq, nc, device=dev, dtype=torch.float32)
        boxes = torch.empty(B, nq, 4, device=dev, dtype=torch.float32)
        aux = None
        res = {"pred_logits": logits, "pred_boxes": boxes}
        if want_aux:
            aux = AuxOut()
            al = torch.empty(nl - 1, B, nq, nc, device=dev, dtype=torch.float32)
            ab = torch.empty(nl - 1, B, nq, 4, device=dev, dtype=torch.float32)
            el = torch.empty(B, nq, nc, device=dev, dtype=torch.float32)
            eb = torch.empty(B, nq, 4, device=dev, dtype=torch.float32)
            ti = torch.empty(B, nq, device=dev, dtype=torch.int32)
            aux.aux_logits, aux.aux_boxes, aux.enc_logits, aux.enc_boxes, aux.topk_index = (
                al.data_ptr(), ab.data_ptr(), el.data_ptr(), eb.data_ptr(), ti.data_ptr())
            res["aux_outputs"] = [{"pred_logits": al[i], "pred_boxes": ab[i]} for i in range(nl - 1)]
            res["enc_outputs"] = {"pred_logits": el, "pred_boxes": eb}
            res["topk_index"] = ti
        return res, logits, boxes, aux

    def forward_frames(self, frames, size=None, fit="stretch", short_side=None, max_side=None, want_aux=True, topk_override=None,
                       mean=IMAGENET_MEAN, std=IMAGENET_STD, colorspace=None, dsts=None, want_hidden=False):
        """Raw camera / decoder frames of any size, RGB or NV12 (told apart by their form):
          RGB: a list of CUDA uint8 [h, w, 3] tensors (each its own size; views with packed RGB pixels are fine) or one
            [B, h, w, 3] tensor;
          NV12: a list of (luma [h, w], chroma [ceil(h/2), 2 * ceil(w/2)]) CUDA uint8 pairs (any row stride), of packed
            [3h/2, w] tensors (h, w even), or one packed [B, 3h/2, w] tensor; colorspace= "bt601", "bt709", "bt601_full" or
            "bt709_full" (one, or one per frame) is required, and each pixel is converted to RGB on the device
            (include/lwdetr_b200.h) as the frame is read.
        Every frame is resized on the device (antialiased bilinear, fused into the patch gather) and normalised with mean / std.
        fit="stretch": to `size` = (H, W), default (img_size, img_size).  fit="keep_aspect": to the reference's
        resize(size=short_side, max_size=max_side), frames top-left on the run size (`size`, or run_size of the largest resized
        frame), the rest padded with a mask made on the device (b200.config.frame_sizes).  Source sizes and the frame format
        are not part of the plan: only a new (B, H, W) re-plans.  dsts: explicit (dst_h, dst_w) per frame, each placed
        top-left on the run size `size` (default img_size x img_size) with the padding mask (the crop views of tiled
        detection, b200.config.tile_views); fit / short_side / max_side do not apply then.  Returns the dict of forward(),
        plus "frame_sizes": the (dst_h, dst_w) of each frame, and with want_hidden "hidden": the final decoder layer's
        hidden state [B, num_queries, hidden_dim] in the activation dtype (lwdetr_last_hidden), the rows class_embed reads;
        row q is the feature of query q (the appearance embedding Tracker.update takes)."""
        import torch
        from .config import explicit_frame_sizes, frame_sizes
        fb = Frames(frames, self.device, colorspace)
        if dsts is None:
            (H, W), dsts = frame_sizes(self.cfg, fb.sizes, size, fit, short_side, max_side)
        else:
            if fit != "stretch" or short_side is not None or max_side is not None:
                raise RuntimeError("lwdetr_b200: dsts= gives every frame's size; fit / short_side / max_side do not combine with it")
            (H, W), dsts = explicit_frame_sizes(self.cfg, len(fb.items), dsts, size)
        B = len(fb.items)
        res, logits, boxes, aux = self._outputs(B, self.device, want_aux)
        ov = None
        if topk_override is not None:
            ov = check_topk_override(topk_override, B, self.cfg.num_queries, self.cfg.memory_len_at(H, W), self.device)
        name ="lwdetr_forward_frames_nv12" if fb.nv12 else "lwdetr_forward_frames"
        check(getattr(lib(), name)(self._h, fb.descs(dsts), ctypes.cast(_norm3(mean), _vp), ctypes.cast(_norm3(std), _vp), B, H, W,
                                   ptr(logits), ptr(boxes), ctypes.byref(aux) if aux is not None else None, ptr(ov),
                                   stream_ptr(self.device)), name)
        self._last_inputs = (fb.items, ov, None)    # keep alive until the stream has consumed them
        res["frame_sizes"] = dsts
        if want_hidden:
            hidden = torch.empty(B, self.cfg.num_queries, self.cfg.hidden_dim, device=self.device, dtype=io_dtype(self.dtype))
            check(lib().lwdetr_last_hidden(self._h, ptr(hidden), self.cfg.hidden_dim, stream_ptr(self.device)), "lwdetr_last_hidden")
            res["hidden"] = hidden
        return res

    # ---- debug captures -------------------------------------------------------------------------
    def capture(self, label, numel):
        import torch
        t = torch.empty(int(numel), dtype=torch.float32)
        check(lib().lwdetr_add_capture(self._h, label.encode(), ptr(t), int(numel)), "lwdetr_add_capture")
        self._captures.append((label, t))
        return t

    def capture_results(self):
        out = {}
        for i, (label, t) in enumerate(self._captures):
            n = lib().lwdetr_capture_result(self._h, i)
            out[label] = t[:n] if n >= 0 else None
        return out

    def clear_captures(self):
        lib().lwdetr_clear_captures(self._h)
        self._captures = []

    def ops(self):
        n = lib().lwdetr_num_ops(self._h)
        out = []
        for i in range(n):
            fl, by = ctypes.c_double(), ctypes.c_double()
            lib().lwdetr_op_cost(self._h, i, ctypes.byref(fl), ctypes.byref(by))
            out.append((lib().lwdetr_op_label(self._h, i).decode(), fl.value, by.value))
        return out

    def profile_ops(self, iters=10):
        n = lib().lwdetr_num_ops(self._h)
        ms = (ctypes.c_float * n)()
        check(lib().lwdetr_profile_ops(self._h, iters, ctypes.cast(ms, _vp), stream_ptr()), "lwdetr_profile_ops")
        return [(lab, fl, by, ms[i]) for i, (lab, fl, by) in enumerate(self.ops())]
