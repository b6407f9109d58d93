"""CPU: the C-ABI library loads without a GPU, exports every symbol include/pepper_b200.h declares, and its
compute entry points fail loudly (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "pepper_b200", "csrc")], check=True)
    from pepper_b200 import _lib
    return _lib.lib()


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "pepper_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pb_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported(lib):
    names = declared_symbols()
    assert len(names) >= 35
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_q8_guard_threshold_matches_header():
    src = open(os.path.join(ROOT, "include", "pepper_b200.h")).read()
    m = re.search(r"#define\s+PB_VARIANT_Q8_MAX_GATE_ERR\s+(\S+)", src)
    from pepper_b200 import abi
    assert m and float(m.group(1)) == abi.PB_VARIANT_Q8_MAX_GATE_ERR


def test_param_tables(lib):
    lib.pb_variant_net_param_name.restype = C.c_char_p
    lib.pb_variant_net_param_numel.restype = C.c_int64
    lib.pb_polish_net_param_name.restype = C.c_char_p
    lib.pb_polish_net_param_numel.restype = C.c_int64
    from pepper_b200 import weights
    sv, sp = weights.random_variant_state(0), weights.random_polish_state(0)
    assert sum(int(lib.pb_variant_net_param_numel(i)) for i in range(28)) == 11862019      # SURVEY: 11,862,019 params
    assert sum(int(lib.pb_polish_net_param_numel(i)) for i in range(18)) == 405253         # SURVEY: 405,253 params
    for i in range(28):
        assert sv[lib.pb_variant_net_param_name(i).decode()].size == lib.pb_variant_net_param_numel(i)
    for i in range(18):
        assert sp[lib.pb_polish_net_param_name(i).decode()].size == lib.pb_polish_net_param_numel(i)


def test_no_cpu_fallback(lib):
    if lib.pb_device_count() > 0:
        pytest.skip("GPU present")
    from pepper_b200 import _lib
    from pepper_b200.variant import VariantEncoder
    with pytest.raises(_lib.PepperB200Error):
        VariantEncoder(0)
    h = C.c_void_p()
    assert lib.pb_polish_encoder_create(C.byref(h), 0) == -2
    lib.pb_last_error.restype = C.c_char_p
    assert b"no CPU fallback" in lib.pb_last_error()


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pepper_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), (dirpath, f)
                assert "liboracle" not in src and "oracle/_ref" not in src, (dirpath, f)


def test_synth_workload_shapes():
    from pepper_b200 import synth
    reads, regions = synth.make_variant_workload(2, 3000, 20, synth.ONT, seed=1)
    assert regions.genomic_bases() == 6000
    assert regions.table[0, 3] == regions.table[1, 2]            # adjacent intervals share their boundary
    r2, g2 = synth.tile_workload(reads, regions, 3)
    assert g2.n_regions == 6 and r2.n_reads == 3 * reads.n_reads and r2.n_bases == 3 * reads.n_bases
    assert np.array_equal(r2.codes()[:reads.n_bases], reads.codes())
