"""The iq_format field of the decoder, cell-search and tracker configurations (no GPU needed): an unknown format is refused by name before any
device is looked for, the three known ones get as far as the device; the field takes the first reserved word, so no struct changed size or the
offset of another field; and every function the headers declare is still exported after the sample pointers became const void *."""
import ctypes as C
import os
import subprocess

import pytest

from ltesniffer_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu():
    import torch
    return torch.cuda.is_available()


def _cfgs(fmt):
    return [("ltephy_create", "ltephy_destroy", capi.Cfg(nof_prb=25, nof_ports=1, cell_id=1, nof_rx=1, max_subframes=1, iq_format=fmt)),
            ("ltephy_sync_create", "ltephy_sync_destroy", capi.SyncCfg(symbol_sz=512, nof_rx=1, max_samples=76 * 512, iq_format=fmt)),
            ("ltephy_track_create", "ltephy_track_destroy", capi.TrackCfg(symbol_sz=512, nof_rx=1, pci=1, max_subframes=10, iq_format=fmt))]


@pytest.mark.parametrize("fmt", [3, 0xFFFFFFFF])
def test_unknown_format_is_refused_by_name(phylib, fmt):
    L = capi.load_library()
    for create, _, cfg in _cfgs(fmt):
        h = C.c_void_p()
        assert getattr(L, create)(C.byref(cfg), C.byref(h)) == -2, create
        assert b"iq_format" in L.ltephy_last_error(), (create, L.ltephy_last_error())
        assert not h.value


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_known_formats_reach_the_device(phylib, fmt):
    L = capi.load_library()
    gpu = _gpu()
    for create, destroy, cfg in _cfgs(fmt):
        h = C.c_void_p()
        rc = getattr(L, create)(C.byref(cfg), C.byref(h))
        if gpu:
            assert rc == 0, (create, L.ltephy_last_error())
            getattr(L, destroy)(h)
        else:
            assert rc == -1 and b"no CUDA device" in L.ltephy_last_error(), (create, rc, L.ltephy_last_error())


def test_struct_layouts_are_unchanged(tmp_path):
    """the binding's structs against the C header: sizes as before the field, and iq_format where the first reserved word was"""
    assert (C.sizeof(capi.Cfg), C.sizeof(capi.SyncCfg), C.sizeof(capi.TrackCfg)) == (64, 40, 64)
    assert (capi.Cfg.iq_format.offset, capi.SyncCfg.iq_format.offset, capi.TrackCfg.iq_format.offset) == (52, 20, 44)
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ltephy_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %u %u %u", sizeof(ltephy_cfg_t), sizeof(ltephy_sync_cfg_t), sizeof(ltephy_track_cfg_t),\n'
                   '  offsetof(ltephy_cfg_t, iq_format), offsetof(ltephy_sync_cfg_t, iq_format), offsetof(ltephy_track_cfg_t, iq_format),\n'
                   '  LTEPHY_IQ_CF32, LTEPHY_IQ_SC16, LTEPHY_IQ_SC8); return 0; }\n')
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", exe, str(src)], check=True)
    got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [64, 40, 64, 52, 20, 44, 0, 1, 2]
    assert capi.IQ_FORMATS == {"cf32": 0, "sc16": 1, "sc8": 2}


@pytest.mark.parametrize("header", ["ltephy_b200.h", "ltephy_search.h", "ltephy_sinks.h", "ltephy_shard.h"])
def test_every_declared_function_is_exported(phylib, header):
    from test_capi_exports import declared_functions
    names = declared_functions(header)
    assert names and not [n for n in names if not hasattr(phylib, n)]


def test_float_callers_still_compile(tmp_path):
    """a C++ caller that hands the library float pointers, as every caller did before the prototypes took const void *, compiles unchanged"""
    src = tmp_path / "caller.cpp"
    src.write_text('#include "ltephy_search.h"\n'
                   'int f(ltephy_t* h, ltephy_search_t* s, ltephy_sync_t* y, ltephy_track_t* t, const float* x, const uint32_t* tti) {\n'
                   '  ltephy_cell_t c[3]; ltephy_track_out_t o; const void* u;\n'
                   '  return ltephy_submit_iq(h, x, tti, 1) + ltephy_submit_ul(h, x, tti, 1, nullptr, 0) + ltephy_cell_search(y, x, 1, c) +\n'
                   '         ltephy_track_push(t, x, 0, 1, &o) + ltephy_track_push_ul(t, x, x, 0, 1, &o, &u) +\n'
                   '         ltephy_decode_subframes(h, s, x, tti, 1, LTEPHY_SEQ_NONE, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, 0); }\n')
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-c", "-I" + os.path.join(ROOT, "include"), "-o", str(tmp_path / "caller.o"), str(src)],
                   check=True)
