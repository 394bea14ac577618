"""CPU checks of the C-ABI: the library loads without a GPU, exports every declared symbol,
and its wl_config layout matches the header the oracle was compiled against."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_library_loads_and_exports_all_header_symbols():
    import wheeledlab_b200 as wl
    header = (ROOT / "include" / "wheeledlab_b200.h").read_text()
    declared = set(re.findall(r"\b(wl_[a-z_0-9]+)\s*\(", header))
    declared -= {"wl_sim"}
    assert declared, "no declarations parsed"
    for sym in sorted(declared):
        assert hasattr(wl.lib, sym), f"{sym} declared in include/wheeledlab_b200.h but not exported"
    from wheeledlab_b200._lib import EXPORTED_SYMBOLS
    assert declared == set(EXPORTED_SYMBOLS)


def test_step_launch_info_rejects_a_null_handle():
    import wheeledlab_b200 as wl
    v, k, s, th = C.c_int32(-7), C.c_uint32(7), C.c_int32(-7), C.c_int32(-7)
    assert wl.lib.wl_step_launch_info(None, C.byref(v), C.byref(k), C.byref(s), C.byref(th)) < 0
    assert b"wl_step_launch_info" in wl.lib.wl_last_error()
    assert (v.value, k.value, s.value, th.value) == (-7, 7, -7, -7), "outputs written on failure"


def test_config_layout_matches_oracle_header():
    import wheeledlab_b200 as wl
    from oracle_lib import get_lib
    assert wl.lib.wl_config_describe().decode() == get_lib().wlo_config_describe().decode()
    assert wl.lib.wl_config_sizeof() == C.sizeof(wl.WlConfig)
    assert C.sizeof(wl.WlConfig) < 4000, "wl_config is passed as a __grid_constant__ kernel parameter (<4 KB)"


def test_state_bytes_and_alignment():
    import wheeledlab_b200 as wl
    for n in (1, 33, 4096):
        off = wl.lib.wl_globals_offset(n)
        assert off % 256 == 0 and off >= 14 * n * 16
        assert wl.lib.wl_state_bytes(n) >= off + 160


def test_build_targets_sm90a():
    import subprocess
    import wheeledlab_b200 as wl
    assert b"sm_90a" in wl.lib.wl_build_info()
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", str(wl.LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_no_cuda_device_fails_loudly():
    import torch
    import wheeledlab_b200 as wl
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(wl.WlError):
        wl.WheeledSim(wl.drift_task(num_envs=4), "cuda:0")
    with pytest.raises(wl.WlError):
        wl.WheeledSim(wl.drift_task(num_envs=4), "cpu")


def test_product_never_imports_oracle():
    pkg = ROOT / "wheeledlab_b200"
    for f in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.cuh")):
        txt = f.read_text()
        assert "oracle" not in txt.replace("the oracle", "").replace("CPU oracle", "").replace("oracle/wl_oracle.c", "").replace("build_oracle", "").replace('"oracle"', "").replace("oracle's", "") or f.name == "build.py", f


def test_plain_c_host_example_builds_against_the_abi(tmp_path):
    """examples/c_host: a gcc program that includes only include/wheeledlab_b200.h and links the in-tree .so + libcudart
    (no compute here: it needs a GPU to run; tests/test_gpu_parity.py runs it)."""
    import shutil
    import subprocess
    root = Path(__file__).resolve().parent.parent
    if not Path("/usr/local/cuda/include/cuda_runtime_api.h").exists():
        pytest.skip("CUDA toolkit headers not present")
    ex = root / "examples" / "c_host"
    subprocess.run(["make", "-C", str(ex), "clean"], check=True, stdout=subprocess.DEVNULL)
    subprocess.run(["make", "-C", str(ex), "CC=" + (shutil.which("gcc", path="/usr/bin") or "gcc")], check=True, stdout=subprocess.DEVNULL)
    assert (ex / "wl_c_host").exists()
    from wheeledlab_b200.dump_config import dump
    from wheeledlab_b200._lib import WlConfig
    import ctypes as C
    assert dump("drift", 64, str(tmp_path / "cfg.bin")) == C.sizeof(WlConfig)


def test_every_exported_symbol_is_documented_in_integration_md():
    """INTEGRATION.md section 3 lists every entry point of the C-ABI with the reference interface it stands for."""
    from wheeledlab_b200._lib import EXPORTED_SYMBOLS
    doc = (ROOT / "INTEGRATION.md").read_text()
    missing = [s for s in EXPORTED_SYMBOLS if s not in doc]
    assert not missing, f"undocumented entry points: {missing}"
