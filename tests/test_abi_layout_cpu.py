"""The ctypes binding against include/lwdetr_b200.h as the host C compiler lays it out: every struct's size and field
offsets, and every struct field and prototype the header declares, so that a binding that drifts from the header fails
here and not by a C call reading past a short struct on the GPU."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")

# each struct of the header and the name capi binds it to
PUBLIC = {"lwdetr_gemm_args": "GemmArgs", "lwdetr_layernorm_args": "LayerNormArgs", "lwdetr_attention_args": "AttentionArgs",
          "lwdetr_tile_view": "TileViewStruct", "lwdetr_track_params": "TrackParams", "lwdetr_track_record": "TrackRecord",
          "lwdetr_reid_params": "ReidParams", "lwdetr_gmc_params": "GmcParams", "lwdetr_flow_params": "FlowParams",
          "lwdetr_zones_params": "ZonesParams", "lwdetr_zone_record": "ZoneRecord", "lwdetr_config": "ConfigStruct",
          "lwdetr_aux_out": "AuxOut", "lwdetr_input": "InputDesc", "lwdetr_frame": "FrameStruct", "lwdetr_frame_nv12": "FrameNV12Struct"}


def _header():
    with open(os.path.join(INCLUDE, "lwdetr_b200.h")) as f:
        return re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)


def test_struct_sizes_and_offsets_match_the_c_compiler(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "no host C compiler on PATH"
    want, prints = {}, []
    for c, py in PUBLIC.items():
        S = getattr(capi, py)
        want[c] = ctypes.sizeof(S)
        prints.append('printf("%s %%zu\\n", sizeof(%s));' % (c, c))
        for f, _ in S._fields_:
            want[c + "." + f] = getattr(S, f).offset
            prints.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (c, f, c, f))
    src = tmp_path / "abi.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"lwdetr_b200.h\"\nint main(void) {\n  %s\n  return 0;\n}\n"
                   % "\n  ".join(prints))
    exe = tmp_path / "abi"
    subprocess.run([cc, "-std=c99", "-I", INCLUDE, str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert {k: int(v) for k, v in (line.split() for line in out.splitlines())} == want


def test_binding_covers_every_struct_field_and_prototype():
    hdr = _header()
    bodies = {name: body for body, name in re.findall(r"typedef\s+struct\s*\{([^}]*)\}\s*(\w+)\s*;", hdr)}
    assert set(bodies) == set(PUBLIC)
    for c, body in bodies.items():
        declared = re.findall(r"(\w+)\s*(?:\[\d+\])?\s*[,;]", body)
        assert [f for f, _ in getattr(capi, PUBLIC[c])._fields_] == declared, c
    protos = dict(re.findall(r"LWDETR_API[^;(]*?\b(lwdetr_\w+)\s*\(([^)]*)\)", hdr))
    assert set(protos) == set(capi._SIGNATURES)
    for name, params in protos.items():
        params = [] if params.strip() == "void" else params.split(",")
        argtypes = capi._SIGNATURES[name][1]
        assert len(argtypes) == len(params), name
        assert [t in (ctypes.c_void_p, ctypes.c_char_p) for t in argtypes] == ["*" in p or "[" in p for p in params], name


@pytest.mark.parametrize("decl, named", [
    ("LWDETR_API unsigned lwdetr_x(int a);", "`unsigned` (lwdetr_x)"),
    ("LWDETR_API int lwdetr_x(long a);", "long a"),
    ("LWDETR_API int (*lwdetr_x)(int a);", "(*lwdetr_x)"),
    ("typedef struct { int32_t a; long b; } lwdetr_y;", "long b"),
    ("typedef struct { int32_t* a[2]; } lwdetr_y;", "a[2]"),
    ("typedef struct { struct { int32_t a; } in; } lwdetr_y;", "struct { int32_t a"),
    ("typedef int32_t lwdetr_z;", "typedef int32_t lwdetr_z"),
])
def test_header_reader_refuses_what_it_does_not_know(tmp_path, decl, named):
    hdr = tmp_path / "h.h"
    hdr.write_text("/* a comment; with a semicolon */\n#define LWDETR_API x\nLWDETR_API int lwdetr_ok(const char* s, int n[2]);\n" + decl + "\n")
    with pytest.raises(RuntimeError, match=re.escape(named)):
        capi._read_header(str(hdr))
