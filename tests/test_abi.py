"""CPU: the C-ABI library builds, loads and exports every symbol include/femasr_b200.h declares;
without a GPU the product path fails loudly instead of falling back."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "femasr_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(femasr_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(built_lib):
    from femasr_b200 import lib
    names = header_symbols()
    assert len(names) >= 30
    dll = ctypes.CDLL(built_lib)
    for n in names:
        assert hasattr(dll, n), f"{n} declared in the header but not exported"
    assert sorted(lib.SIGNATURES) == names, "femasr_b200/lib.py SIGNATURES out of sync with the header"
    assert lib.load().femasr_abi_version() == lib.ABI_VERSION == 4


WRITABLE_DEVICE_SECTIONS = (".nv.global", ".nv.global.init", ".nv.constant3")
_HEX = r"(?:0x)?[0-9a-f]+"
_SECTION_ROW = re.compile(rf"^\s*({_HEX})\s+{_HEX}\s+{_HEX}\s+{_HEX}\s+{_HEX}\s+[A-Z_]+\s+{_HEX}\s+{_HEX}\s+{_HEX}\s+(\S+)$")
_SYMBOL_ROW = re.compile(rf"^\s*{_HEX}\s+{_HEX}\s+{_HEX}\s+({_HEX})\s+{_HEX}\s+({_HEX})\s+(\S+)$")


def device_globals(elf_dump):
    """{symbol: section} of every symbol `cuobjdump -elf` lists in a writable library-global device section (__device__
    variables land in .nv.global / .nv.global.init, __constant__ ones in .nv.constant3), over every cubin in the dump."""
    found = {}
    for cubin in elf_dump.split("Fatbin elf code:")[1:]:
        sections, in_symtab = {}, False
        for line in cubin.splitlines():
            if line.startswith(".section"):
                in_symtab = line.split()[1] == ".symtab"
            elif not in_symtab and (m := _SECTION_ROW.match(line)):       # Index Offset Size ES Align Type Flags Link Info Name
                sections[int(m[1], 16)] = m[2]
            elif in_symtab and (m := _SYMBOL_ROW.match(line)):            # index value size info other shndx name
                sec = sections.get(int(m[2], 16), "")
                if sec in WRITABLE_DEVICE_SECTIONS and (int(m[1], 16) & 0xF) != 3:   # STT_SECTION rows name the section
                    found[m[3]] = sec
    return found


def test_library_has_no_device_globals(built_lib):
    """Engines on separate streams or host threads of one device run concurrently, so no kernel may keep its operands in
    library-global device memory: every weight travels through the handle's own buffers.  A __device__ or __constant__
    variable in the library is state shared by every engine in the process."""
    from femasr_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found beside nvcc")
    dump = subprocess.run([cuobjdump, "-elf", built_lib], check=True, capture_output=True, text=True).stdout
    assert dump.count("Fatbin elf code:") >= len(build.sources()), "cuobjdump listed fewer cubins than sources"
    found = device_globals(dump)
    assert not found, "library-global device variables: " + ", ".join(f"{k} ({v})" for k, v in sorted(found.items()))


def test_argument_validation_without_gpu(built_lib):
    from femasr_b200 import lib
    L = lib.load()
    a = lib.IgemmArgs()
    assert L.femasr_igemm_simt(ctypes.byref(a), None) == -1
    assert b"null" in L.femasr_last_error()
    h = ctypes.c_void_p()
    cfg = lib.NetConfig(3, 1024, 256, 3, 1, 1, 0)
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    cfg = lib.NetConfig(1, 1024, 256, 3, 1, 1, 1)                 # HQ autoencoder stage
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    need = ctypes.c_size_t()
    assert L.femasr_net_workspace_bytes(h, 2, 64, 96, ctypes.byref(need)) == 0 and need.value > 0
    assert L.femasr_net_workspace_bytes(h, 2, 60, 96, ctypes.byref(need)) == -1
    L.femasr_net_destroy(h)
    cfg = lib.NetConfig(4, 1024, 256, 3, 1, 1, 0)
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    need = ctypes.c_size_t()
    # 40x40: Swin stage 20x20 is not a multiple of the 8x8 window -> the reference raises in window_partition
    assert L.femasr_net_workspace_bytes(h, 1, 40, 40, ctypes.byref(need)) == -1
    assert L.femasr_net_workspace_bytes(h, 32, 128, 128, ctypes.byref(need)) == 0
    assert 1 << 30 < need.value < 40 << 30
    assert abs(L.femasr_net_flops(h, 1, 128, 128) / 1e9 - 754.53) < 0.01
    assert L.femasr_net_params_complete(h) == -3
    L.femasr_net_destroy(h)
    # multi-scale codebooks: geometry, workspace and the FLOP model follow the extra quantisers
    I3 = ctypes.c_int * 3
    cfg = lib.NetConfig(4, 0, 0, 3, 1, 1, 0, 2, I3(32, 64, 0), I3(1024, 512, 0), I3(256, 128, 0))
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    assert L.femasr_net_workspace_bytes(h, 1, 32, 32, ctypes.byref(need)) == 0 and need.value > 0
    extra = 2.0 * 512 * 128 + 2.0 * 512 * 128 + 2.0 * 9 * (128 + 256) * 256       # before_quant, z.E^T, after_quant at 128x128
    assert abs(L.femasr_net_flops(h, 1, 128, 128) - (754.53e9 + extra * 128 * 128)) < 2e7
    L.femasr_net_destroy(h)
    cfg = lib.NetConfig(4, 0, 0, 3, 1, 1, 0, 2, I3(32, 32, 0), I3(1024, 512, 0), I3(256, 128, 0))
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == -1            # scales must increase


def test_set_poison_range_without_gpu(built_lib):
    """femasr_net_set_poison takes -1 (off) or one byte value, on every handle kind, and needs no device."""
    from femasr_b200 import lib
    L = lib.load()
    assert L.femasr_net_set_poison(None, 0) == -1
    for create, cfg in ((L.femasr_net_create, lib.NetConfig(4, 1024, 256, 3, 1, 1, 1)),
                        (L.femasr_disc_create, lib.DiscConfig(3, 64, 1, 0)), (L.femasr_lpips_create, lib.LpipsConfig(1, 1))):
        h = ctypes.c_void_p()
        assert create(ctypes.byref(cfg), ctypes.byref(h)) == 0
        try:
            for bad in (256, -2, 1 << 30, -(1 << 30)):
                assert L.femasr_net_set_poison(h, bad) == -1
                assert b"set_poison" in L.femasr_last_error()
            for good in (0, 0x41, 255, -1):
                assert L.femasr_net_set_poison(h, good) == 0
        finally:
            L.femasr_net_destroy(h)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(built_lib):
    from basicsr.archs.femasr_arch import FeMaSRNet
    from femasr_b200.lib import FemasrError
    net = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=4).eval()
    with pytest.raises(FemasrError):
        net.test(torch.rand(1, 3, 32, 32))
    with pytest.raises(FemasrError):
        net(torch.rand(1, 3, 32, 32))


def test_unsupported_configs_raise():
    from basicsr.archs.femasr_arch import FeMaSRNet
    with pytest.raises(NotImplementedError):
        FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, norm_type="bn")
    with pytest.raises(NotImplementedError):
        FeMaSRNet(codebook_params=[[16, 1024, 256]], LQ_stage=True)               # first codebook must sit at 32
    with pytest.raises(NotImplementedError):
        FeMaSRNet(codebook_params=[[32, 1024, 256], [256, 512, 64]], LQ_stage=True)    # no decoder level at 256
    with pytest.raises(NotImplementedError):
        FeMaSRNet(codebook_params=[[32, 1000, 256]], LQ_stage=True)                # n_e / e_dim: multiples of 64
    ms = FeMaSRNet(codebook_params=[[32, 1024, 256], [64, 512, 128]], LQ_stage=True)   # multi-scale codebooks
    sd = ms.state_dict()
    assert tuple(sd["before_quant_group.1.weight"].shape) == (128, 512, 1, 1)      # femasr_arch.py:292,297
    assert tuple(sd["after_quant_group.1.conv.weight"].shape) == (256, 256 + 128, 3, 3)     # :293-294,298
    assert tuple(sd["quantize_group.1.embedding.weight"].shape) == (512, 128)
    hq = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=False, scale_factor=4)    # HQ stage: scale forced to 1
    assert hq.scale_factor == 1 and not any("swin" in k for k in hq.state_dict())


def test_module_copy_and_checkpoint_roundtrip(tmp_path):
    # copies dropping the native handle: tests/test_engine_module.py
    from basicsr.archs.femasr_arch import FeMaSRNet
    net = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=2).eval()
    path = tmp_path / "w.pth"
    torch.save({"params": net.state_dict()}, path)            # the reference's checkpoint format (base_model.py:212-239)
    other = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=2)
    missing = other.load_state_dict(torch.load(path)["params"], strict=False)
    assert not missing.missing_keys and not missing.unexpected_keys
    for k, v in net.state_dict().items():
        assert torch.equal(v, other.state_dict()[k])


def test_graft_entry_build_runs():
    """The driver's build check: __graft_entry__.build() must compile the library and import the package (CPU only)."""
    import importlib
    ge = importlib.import_module("__graft_entry__")
    ge.build()
