"""The C-ABI library loads on a machine without a GPU and exports every symbol declared in include/*.h
(no compute call is made here). Also checks that there is no silent CPU path: creating a context without
a device fails with HNB_ERR_NO_DEVICE."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    names = []
    for h in sorted((ROOT / "include").glob("*.h")):
        for m in re.finditer(r"HNB_API\s+[^;(]*?\b(hnb_[a-z0-9_]+)\s*\(", h.read_text()):
            names.append((h.name, m.group(1)))
    return names


def test_headers_declare_something():
    names = [n for _, n in _declared()]
    assert len(names) >= 70
    for must in ("hnb_ctx_create", "hnb_simulate", "hnb_slab_create", "hnb_effect_compile", "hnb_asset_generate", "hnb_module_binary",
                 "hnb_read_tile_size"):  # the tests' proof that HNB_TILE_CHUNKS reached the update launch
        assert must in names


@pytest.mark.parametrize("header,name", _declared())
def test_symbol_exported(header, name):
    from bevy_hanabi_b200 import _native as N
    assert hasattr(N.lib, name), f"{name} (declared in include/{header}) is not exported by libhanabi_b200.so"


def test_python_binding_covers_every_symbol():
    from bevy_hanabi_b200 import _native as N
    from bevy_hanabi_b200 import graph as G
    from bevy_hanabi_b200 import cache as K
    from bevy_hanabi_b200 import spawn as S
    bound = set(N.SIGNATURES) | set(G.GRAPH_SIGNATURES) | set(S.SPAWN_SIGNATURES) | set(K.CACHE_SIGNATURES)
    declared = {n for _, n in _declared()}
    assert declared <= bound, f"unbound: {sorted(declared - bound)}"


def test_struct_sizes_match_reference_layouts():
    from bevy_hanabi_b200 import _native as N
    assert C.sizeof(N.Spawner) == 128          # GpuSpawnerParams
    assert C.sizeof(N.EffectMetadata) == 60    # GpuEffectMetadata
    assert C.sizeof(N.BatchInfo) == 24         # GpuBatchInfo
    assert C.sizeof(N.SimParams) == 28         # GpuSimParams
    assert C.sizeof(N.DrawIndexedIndirectArgs) == 20
    assert C.sizeof(N.DispatchIndirectArgs) == 12
    assert C.sizeof(N.IndirectIndex) == 12
    assert C.sizeof(N.ChildInfo) == 8
    assert N.Spawner.spawn.offset == 96 and N.Spawner.seed.offset == 100 and N.Spawner.slab_offset.offset == 116
    assert N.EffectMetadata.particle_counter.offset == 56 and N.EffectMetadata.indirect_write_index.offset == 16


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from bevy_hanabi_b200 import _native as N
    h = C.c_void_p()
    rc = N.lib.hnb_ctx_create(0, 0, C.byref(h))
    assert rc == N.HNB_ERR_NO_DEVICE
    assert "no CPU fallback" in N.last_error() or "driver" in N.last_error().lower()
    assert not h.value


def test_product_does_not_import_oracle():
    """The product package must never reach into oracle/ (test infrastructure only)."""
    for py in (ROOT / "bevy_hanabi_b200").rglob("*.py"):
        txt = py.read_text()
        assert "import oracle" not in txt and "from oracle" not in txt, py
    for src in (ROOT / "bevy_hanabi_b200" / "csrc").rglob("*"):
        if src.is_file() and src.suffix in (".cpp", ".cu", ".cuh", ".h"):
            assert "vfx_oracle" not in src.read_text(), src
