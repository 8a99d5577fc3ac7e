"""The C-ABI library loads (no GPU needed) and exports every function include/*.h declares; creation fails
loudly without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re
import pytest
from ltesniffer_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(ltephy_[a-z0-9_]+)\s*\(", txt)))


@pytest.mark.parametrize("header", ["ltephy_b200.h", "ltephy_search.h", "ltephy_sinks.h", "ltephy_shard.h"])
def test_every_declared_symbol_is_exported(phylib, header):
    names = declared_functions(header)
    assert len(names) >= 7
    missing = [n for n in names if not hasattr(phylib, n)]
    assert not missing, "declared in include/%s but not exported: %s" % (header, missing)


def test_create_fails_loudly_without_gpu(phylib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        capi.LtePhy(100, 1, 1, 1)


def test_invalid_inputs_are_rejected(phylib):
    h = C.c_void_p()
    cfg = capi.Cfg(nof_prb=6, nof_ports=1, cell_id=0, nof_rx=1, max_subframes=1)
    assert phylib.ltephy_create(C.byref(cfg), C.byref(h)) == -2   # LTEPHY_ERROR_INVALID_INPUTS (falcon_pdcch.c:121 convention)
    assert phylib.ltephy_create(None, C.byref(h)) == -2
    # the front end's grids put the subframe on gridDim.y / z (at most 65 535): refused before any device is looked for
    for ms in (65536, 100000, 0xFFFFFFFF):
        cfg = capi.Cfg(nof_prb=25, nof_ports=1, cell_id=0, nof_rx=1, max_subframes=ms)
        assert phylib.ltephy_create(C.byref(cfg), C.byref(h)) == -2
        assert b"max_subframes" in phylib.ltephy_last_error()


def test_srsran_compat_shim_exports(phylib):
    """tier-2 library: loads on top of libltephy_b200.so and exports every function the srsRAN-compatible header tree compat/srsran declares"""
    from ltesniffer_b200 import build
    assert os.path.exists(build.COMPAT_OUT)
    lib = C.CDLL(build.COMPAT_OUT)
    names = set()
    for r, _, fs in os.walk(os.path.join(ROOT, "compat", "srsran")):
        for f in fs:
            txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(r, f)).read(), flags=re.S)
            txt = re.sub(r"//.*", "", txt)
            names |= set(re.findall(r"\b(srsran_[a-z0-9_]+)\s*\(", txt))
    must = {"srsran_ue_dl_init", "srsran_ue_dl_set_cell", "srsran_ue_dl_free", "srsran_ue_dl_decode_fft_estimate", "srsran_pdcch_dci_decode",
            "srsran_ue_dl_decode_pdsch", "srsran_enb_ul_init", "srsran_enb_ul_set_cell", "srsran_enb_ul_fft", "srsran_chest_ul_estimate_pusch",
            "srsran_pusch_decode", "srsran_softbuffer_rx_init", "srsran_softbuffer_rx_free", "srsran_softbuffer_rx_reset_tbs", "srsran_dci_format_sizeof",
            "srsran_dci_msg_unpack_pdsch", "srsran_dci_msg_unpack_pusch", "srsran_ra_dl_grant_to_grant_prb_allocation", "srsran_ra_tbs_from_idx",
            "srsran_ra_ul_dci_to_grant", "srsran_pdcch_ue_locations_ncce", "srsran_pdcch_common_locations_ncce"}
    assert must <= names and len(names) >= 100
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, "declared in compat/srsran but not exported: %s" % missing
    assert hasattr(lib, "ltephy_compat_inject") and hasattr(lib, "ltephy_compat_phy")
