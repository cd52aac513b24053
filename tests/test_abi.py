"""CPU-side checks of the drop-in boundary: the shared library loads, exports every function that
include/stx.h declares, and the ctypes binding declares exactly those (no compute call is made)."""
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def header_functions():
    text = (ROOT / "include" / "stx.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(stx_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from stoix_b200 import _lib

    path = _lib.library_path()
    if not path.exists():
        from stoix_b200.build import build_library

        build_library()
    lib = ctypes.CDLL(str(path))
    names = header_functions()
    assert len(names) >= 20
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/stx.h but not exported"


def test_binding_matches_header():
    from stoix_b200 import _lib

    assert sorted(_lib.declared_symbols()) == header_functions()
    assert _lib.load().stx_version() == 100


def test_struct_layouts_match_c():
    from stoix_b200 import _lib

    assert ctypes.sizeof(_lib.StxMlp) == (4 + 8 * 4 + 4) + 8 + 8 + 4 + 4  # n_layers, sizes[8], pad to 8, two pointers, two ints
    assert ctypes.sizeof(_lib.StxAdamSeg) == 24
    assert ctypes.sizeof(_lib.StxAdamHyper) == 32
    assert ctypes.sizeof(_lib.StxPpoHyper) == 32
    assert ctypes.sizeof(_lib.StxPpoBatch) == 72
    assert ctypes.sizeof(_lib.StxReplay) == 6 * 8 + 8 + 4 + 4


def test_ops_refuse_cpu_tensors_and_missing_library(monkeypatch, tmp_path):
    import torch

    from stoix_b200 import _lib, ops

    with pytest.raises(_lib.StxError):
        ops.make_permutation(8, 0, 0, out=torch.zeros(8, dtype=torch.int32))
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "_LIB_PATH", tmp_path / "missing.so")
    with pytest.raises(_lib.StxError, match="no CPU or PyTorch fallback"):
        _lib.load()


def test_config_layer_and_shape_derivation():
    from stoix_b200.config import compose
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_ppo", ["env=synthetic/box", "arch.total_num_envs=32768", "arch.total_timesteps=41943040", "arch.num_evaluation=5"])
    cfg.num_devices = 8
    cfg = check_total_timesteps(cfg, quiet=True)
    assert (cfg.arch.num_envs, cfg.arch.num_updates, cfg.arch.num_updates_per_eval) == (4096, 10, 2)
    assert cfg.network.actor_network.pre_torso._target_ == "stoix.networks.torso.MLPTorso"
    with pytest.raises(AssertionError):
        cfg.arch.total_num_envs = 1001
        check_total_timesteps(cfg, quiet=True)
