"""Drop-in for the reference's compiled pybind11 module `MultiScaleDeformableAttention`
(models/ops/setup.py:53, src/vision.cpp:13-16): same module name, same two functions, same argument order, so
models/ops/functions/ms_deform_attn_func.py:23 (`import MultiScaleDeformableAttention as MSDA`) binds to the CUDA-native
kernels without any edit when lw-detr_b200/ precedes the reference tree on PYTHONPATH.

    ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step) -> output
    ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step)
        -> [grad_value, grad_sampling_loc, grad_attn_weight]

Both go through the C ABI (include/lwdetr_b200.h: lwdetr_ms_deform_attn_forward / _backward).  Like the reference
op (ms_deform_attn.h:19-35) they raise RuntimeError for CPU tensors ("Not implemented on the CPU") and for
non-contiguous tensors; unlike it the forward also accepts float16 / bfloat16, and float64 inputs are computed in
float32 (the H100's fp64 rate is no use to a gather) and returned as float64."""
import torch

from b200 import capi


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
    if value.dtype == torch.float64:
        out = capi.ms_deform_attn_forward(value.float(), spatial_shapes, level_start_index, sampling_loc.float(), attn_weight.float(), im2col_step)
        return out.double()
    return capi.ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step):
    dt = value.dtype
    f = lambda t: t.float().contiguous()
    gv, gl, ga = capi.ms_deform_attn_backward(f(value), spatial_shapes, level_start_index, f(sampling_loc), f(attn_weight), f(grad_output), im2col_step)
    return [gv.to(dt), gl.to(dt), ga.to(dt)]
