"""CPU: the engine's plan - status, workspace bytes (with and without the semantic loss), decode workspace bytes and the
FLOP count of one forward - for a grid of configurations, and the status, workspace bytes and FLOP count of the
discriminator and LPIPS handles.  The create calls and these queries never touch a device, so the tables pin the
host-side graphs (arena allocation order, launch list, taps that change the plan) without a GPU."""
import ctypes

import pytest

from femasr_b200 import lib

SHAPES = ((1, 64, 64), (4, 128, 128), (2, 96, 160), (1, 40, 40), (2, 60, 96), (0, 64, 64))
DIV = {4: 2, 2: 4, 1: 8}          # input size / latent (decoder level 0) size

# name -> (scale_factor, codebook_params, enable_semantic, in_conv tap registered)
CONFIGS = {
    "x4_e256": (4, [[32, 1024, 256]], False, False),
    "x4_e512": (4, [[32, 1024, 512]], False, False),
    "x2_e256": (2, [[32, 1024, 256]], False, False),
    "x2_e512": (2, [[32, 1024, 512]], False, False),
    "hq_e256": (1, [[32, 1024, 256]], False, False),
    "hq_e512": (1, [[32, 1024, 512]], False, False),
    "x4_cb2": (4, [[32, 1024, 256], [64, 512, 128]], False, False),
    "x2_cb3": (2, [[32, 1024, 512], [64, 512, 256], [128, 256, 128]], False, False),
    "hq_cb2": (1, [[32, 1024, 512], [128, 512, 256]], False, False),
    "hq_e512_sem": (1, [[32, 1024, 512]], True, False),
    "x4_e512_sem": (4, [[32, 1024, 512]], True, False),       # the semantic loss does not exist in the LQ stage
    "x4_e256_tap": (4, [[32, 1024, 256]], False, True),
}


def plan(L, name, gemm_path):
    """{"BxHxW": [status, bytes, sem status, sem bytes, decode bytes, flops]} (bytes / flops None where not defined)."""
    scale, cbs, sem, tap = CONFIGS[name]
    I3 = ctypes.c_int * 3
    pad = lambda v: I3(*(v + [0] * (3 - len(v))))
    cfg = lib.NetConfig(scale, cbs[0][1], cbs[0][2], 3, 1, 1, gemm_path, len(cbs), pad([c[0] for c in cbs]),
                        pad([c[1] for c in cbs]), pad([c[2] for c in cbs]))
    h = ctypes.c_void_p()
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    try:
        if sem:
            assert L.femasr_net_enable_semantic(h) == 0
        if tap:      # never written in a sizing run; registering it is what changes the plan
            assert L.femasr_net_set_tap(h, b"in_conv", ctypes.c_void_p(1 << 20), 1 << 40) == 0
        out = {}
        for (B, H, W) in SHAPES:
            n, ns, nd = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
            s = L.femasr_net_workspace_bytes(h, B, H, W, ctypes.byref(n))
            s0 = L.femasr_net_workspace_bytes_sem(h, B, H, W, 0, ctypes.byref(ns))
            assert s0 == s and (s or ns.value == n.value)
            ss = L.femasr_net_workspace_bytes_sem(h, B, H, W, 1, ctypes.byref(ns))
            row = [s, n.value if s == 0 else None, ss, ns.value if ss == 0 else None, None, None]
            if s == 0:
                assert L.femasr_net_decode_workspace_bytes(h, B, H // DIV[scale], W // DIV[scale], ctypes.byref(nd)) == 0
                row[4] = nd.value
                row[5] = L.femasr_net_flops(h, B, H, W)
            out[f"{B}x{H}x{W}"] = row
        return out
    finally:
        L.femasr_net_destroy(h)


N = None
# measured with the engine as of the multi-scale codebook / semantic-loss graph; N = not defined (error status)
EXPECTED = {
    "x4_e256/gp0": {
        "1x64x64": [0, 63833344, -3, N, 48234752, 188631506944.0],
        "4x128x128": [0, 1022365952, -3, N, 771752192, 3018128982016.0],
        "2x96x160": [0, 479201536, -3, N, 361758976, 1414747176960.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e256/gp1": {
        "1x64x64": [0, 80610560, -3, N, 65011968, 188631506944.0],
        "4x128x128": [0, 1290801408, -3, N, 1040187648, 3018128982016.0],
        "2x96x160": [0, 605030656, -3, N, 487588096, 1414747176960.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e512/gp0": {
        "1x64x64": [0, 65930496, -3, N, 49283328, 190510555136.0],
        "4x128x128": [0, 1055920384, -3, N, 788529408, 3048193753088.0],
        "2x96x160": [0, 494930176, -3, N, 369623296, 1428840038400.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e512/gp1": {
        "1x64x64": [0, 83756288, -3, N, 66060544, 190510555136.0],
        "4x128x128": [0, 1341133056, -3, N, 1056964864, 3048193753088.0],
        "2x96x160": [0, 628623616, -3, N, 495452416, 1428840038400.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_e256/gp0": {
        "1x64x64": [0, 16515328, -3, N, 12058880, 52618080256.0],
        "4x128x128": [0, 264241408, -3, N, 192938240, 841901719552.0],
        "2x96x160": [0, 123863296, -3, N, 90439936, 394641039360.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_e256/gp1": {
        "1x64x64": [0, 19932416, -3, N, 16253184, 52618080256.0],
        "4x128x128": [0, 318914816, -3, N, 260047104, 841901719552.0],
        "2x96x160": [0, 149491456, -3, N, 121897216, 394641039360.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_e512/gp0": {
        "1x64x64": [0, 17039616, -3, N, 12321024, 53087842304.0],
        "4x128x128": [0, 272630016, -3, N, 197132544, 849417912320.0],
        "2x96x160": [0, 127795456, -3, N, 92406016, 398164254720.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_e512/gp1": {
        "1x64x64": [0, 20718848, -3, N, 16515328, 53087842304.0],
        "4x128x128": [0, 331497728, -3, N, 264241408, 849417912320.0],
        "2x96x160": [0, 155389696, -3, N, 123863296, 398164254720.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e256/gp0": {
        "1x64x64": [0, 3211520, -3, N, 3014912, 8385206272.0],
        "4x128x128": [0, 51380480, -3, N, 48234752, 134169518080.0],
        "2x96x160": [0, 24084736, -3, N, 22610176, 62891765760.0],
        "1x40x40": [0, 1254656, -3, N, 1177856, 3275290624.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e256/gp1": {
        "1x64x64": [0, 4260096, -3, N, 4063488, 8385206272.0],
        "4x128x128": [0, 68157696, -3, N, 65011968, 134169518080.0],
        "2x96x160": [0, 31949056, -3, N, 30474496, 62891765760.0],
        "1x40x40": [0, 1664256, -3, N, 1587456, 3275290624.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e512/gp0": {
        "1x64x64": [0, 3277056, -3, N, 3080448, 8502646784.0],
        "4x128x128": [0, 52429056, -3, N, 49283328, 136048566272.0],
        "2x96x160": [0, 24576256, -3, N, 23101696, 63772569600.0],
        "1x40x40": [0, 1280256, -3, N, 1203456, 3321165824.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e512/gp1": {
        "1x64x64": [0, 4456704, -3, N, 4129024, 8502646784.0],
        "4x128x128": [0, 71303424, -3, N, 66060544, 136048566272.0],
        "2x96x160": [0, 33423616, -3, N, 30966016, 63772569600.0],
        "1x40x40": [0, 1741056, -3, N, 1613056, 3321165824.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_cb2/gp0": {
        "1x64x64": [0, 74319104, -3, N, 48234752, 196953006080.0],
        "4x128x128": [0, 1190138112, -3, N, 771752192, 3151272968192.0],
        "2x96x160": [0, 557844736, -3, N, 361758976, 1477158420480.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_cb2/gp1": {
        "1x64x64": [0, 82707712, -3, N, 65011968, 196953006080.0],
        "4x128x128": [0, 1324355840, -3, N, 1040187648, 3151272968192.0],
        "2x96x160": [0, 620759296, -3, N, 487588096, 1477158420480.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_cb3/gp0": {
        "1x64x64": [0, 23331072, -3, N, 12321024, 61409341440.0],
        "4x128x128": [0, 373293312, -3, N, 197132544, 982561898496.0],
        "2x96x160": [0, 174981376, -3, N, 92406016, 460575498240.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x2_cb3/gp1": {
        "1x64x64": [0, 26518784, -3, N, 16515328, 61409341440.0],
        "4x128x128": [0, 424296704, -3, N, 264241408, 982561898496.0],
        "2x96x160": [0, 198889216, -3, N, 123863296, 460575498240.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_cb2/gp0": {
        "1x64x64": [0, 10453504, -3, N, 3080448, 10717239296.0],
        "4x128x128": [0, 167511296, -3, N, 49283328, 171482046464.0],
        "2x96x160": [0, 78512896, -3, N, 23101696, 80382013440.0],
        "1x40x40": [0, 4076032, -3, N, 1203456, 4186241024.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_cb2/gp1": {
        "1x64x64": [0, 12026624, -3, N, 4129024, 10717239296.0],
        "4x128x128": [0, 192677120, -3, N, 66060544, 171482046464.0],
        "2x96x160": [0, 90309376, -3, N, 30966016, 80382013440.0],
        "1x40x40": [0, 4690688, -3, N, 1613056, 4186241024.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e512_sem/gp0": {
        "1x64x64": [0, 3277056, 0, 3342592, 3080448, 8502646784.0],
        "4x128x128": [0, 52429056, 0, 53477632, 49283328, 136048566272.0],
        "2x96x160": [0, 24576256, 0, 25067776, 23101696, 63772569600.0],
        "1x40x40": [0, 1280256, 0, 1305856, 1203456, 3321165824.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "hq_e512_sem/gp1": {
        "1x64x64": [0, 4456704, 0, 4587776, 4129024, 8502646784.0],
        "4x128x128": [0, 71303424, 0, 73400576, 66060544, 136048566272.0],
        "2x96x160": [0, 33423616, 0, 34406656, 30966016, 63772569600.0],
        "1x40x40": [0, 1741056, 0, 1792256, 1613056, 3321165824.0],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e512_sem/gp0": {
        "1x64x64": [0, 65930496, -1, N, 49283328, 190510555136.0],
        "4x128x128": [0, 1055920384, -1, N, 788529408, 3048193753088.0],
        "2x96x160": [0, 494930176, -1, N, 369623296, 1428840038400.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e512_sem/gp1": {
        "1x64x64": [0, 83756288, -1, N, 66060544, 190510555136.0],
        "4x128x128": [0, 1341133056, -1, N, 1056964864, 3048193753088.0],
        "2x96x160": [0, 628623616, -1, N, 495452416, 1428840038400.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e256_tap/gp0": {
        "1x64x64": [0, 63833344, -3, N, 48234752, 188631506944.0],
        "4x128x128": [0, 1022365952, -3, N, 771752192, 3018128982016.0],
        "2x96x160": [0, 479201536, -3, N, 361758976, 1414747176960.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
    "x4_e256_tap/gp1": {
        "1x64x64": [0, 80480512, -3, N, 65011968, 188631506944.0],
        "4x128x128": [0, 1289756928, -3, N, 1040187648, 3018128982016.0],
        "2x96x160": [0, 604508416, -3, N, 487588096, 1414747176960.0],
        "1x40x40": [-1, N, -1, N, N, N],
        "2x60x96": [-1, N, -1, N, N, N],
        "0x64x64": [-1, N, -1, N, N, N],
    },
}


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_engine_plan(built_lib, name, gemm_path):
    got = plan(lib.load(), name, gemm_path)
    want = EXPECTED[f"{name}/gp{gemm_path}"]
    assert sorted(got) == sorted(want)
    for shape, (s, n, ss, ns, nd, fl) in want.items():
        g = got[shape]
        assert g[:5] == [s, n, ss, ns, nd], (shape, g, want[shape])
        if fl is None:
            assert g[5] is None
        else:
            assert g[5] == pytest.approx(fl, rel=1e-12, abs=0), shape


HEAD_SHAPES = {
    "disc": ((1, 64, 64), (2, 96, 160), (4, 256, 256), (1, 36, 40)),
    "alex": ((1, 31, 31), (2, 67, 93), (8, 256, 256), (1, 30, 64)),
    "vgg": ((1, 32, 48), (2, 64, 96), (8, 256, 256), (1, 24, 64)),
}
# name -> (shape table, skip_connection for the discriminator / net for LPIPS)
HEADS = {"disc_skip": ("disc", 1), "disc_noskip": ("disc", 0), "lpips_alex": ("alex", 0), "lpips_vgg": ("vgg", 1)}


def head_plan(L, name, gemm_path):
    """The discriminator's or LPIPS' plan: {"BxHxW": [status, workspace bytes, flops]} (None where not defined)."""
    kind, arg = HEADS[name]
    h = ctypes.c_void_p()
    if kind == "disc":
        assert L.femasr_disc_create(ctypes.byref(lib.DiscConfig(3, 64, arg, gemm_path)), ctypes.byref(h)) == 0
        ws, flops = L.femasr_disc_workspace_bytes, L.femasr_disc_flops
    else:
        assert L.femasr_lpips_create(ctypes.byref(lib.LpipsConfig(arg, gemm_path)), ctypes.byref(h)) == 0
        ws, flops = L.femasr_lpips_workspace_bytes, L.femasr_lpips_flops
    try:
        out = {}
        for (B, H, W) in HEAD_SHAPES[kind]:
            n = ctypes.c_size_t()
            s = ws(h, B, H, W, ctypes.byref(n))
            out[f"{B}x{H}x{W}"] = [s, n.value if s == 0 else None, flops(h, B, H, W) if s == 0 else None]
        return out
    finally:
        L.femasr_net_destroy(h)


HEAD_EXPECTED = {
    "disc_skip/gp0": {
        "1x64x64": [0, 4194560, 3240099840.0],
        "2x96x160": [0, 31457536, 24300748800.0],
        "4x256x256": [0, 268435712, 207366389760.0],
        "1x36x40": [-1, N, N],
    },
    "disc_skip/gp1": {
        "1x64x64": [0, 4194560, 3240099840.0],
        "2x96x160": [0, 31457536, 24300748800.0],
        "4x256x256": [0, 268435712, 207366389760.0],
        "1x36x40": [-1, N, N],
    },
    "disc_noskip/gp0": {
        "1x64x64": [0, 4194560, 3240099840.0],
        "2x96x160": [0, 31457536, 24300748800.0],
        "4x256x256": [0, 268435712, 207366389760.0],
        "1x36x40": [-1, N, N],
    },
    "disc_noskip/gp1": {
        "1x64x64": [0, 4194560, 3240099840.0],
        "2x96x160": [0, 31457536, 24300748800.0],
        "4x256x256": [0, 268435712, 207366389760.0],
        "1x36x40": [-1, N, N],
    },
    "lpips_alex/gp0": {
        "1x31x31": [0, 176128, 24165120.0],
        "2x67x93": [0, 2523648, 442712064.0],
        "8x256x256": [0, 113799680, 27792070656.0],
        "1x30x64": [-1, N, N],
    },
    "lpips_alex/gp1": {
        "1x31x31": [0, 176128, 24165120.0],
        "2x67x93": [0, 2523648, 442712064.0],
        "8x256x256": [0, 113799680, 27792070656.0],
        "1x30x64": [-1, N, N],
    },
    "lpips_vgg/gp0": {
        "1x32x48": [0, 1573376, 1879179264.0],
        "2x64x96": [0, 12583424, 15033434112.0],
        "8x256x256": [0, 536871424, 641426522112.0],
        "1x24x64": [-1, N, N],
    },
    "lpips_vgg/gp1": {
        "1x32x48": [0, 1573376, 1879179264.0],
        "2x64x96": [0, 12583424, 15033434112.0],
        "8x256x256": [0, 536871424, 641426522112.0],
        "1x24x64": [-1, N, N],
    },
}


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("name", sorted(HEADS))
def test_head_plan(built_lib, name, gemm_path):
    got = head_plan(lib.load(), name, gemm_path)
    assert got == HEAD_EXPECTED[f"{name}/gp{gemm_path}"]


def test_in_conv_tap_changes_the_tensor_core_plan(built_lib):
    """Registering the in_conv tap makes gemm_path 1 run the fp32 in_conv next to the split one."""
    L = lib.load()
    assert plan(L, "x4_e256", 1)["4x128x128"][1] == 1290801408
    assert plan(L, "x4_e256_tap", 1)["4x128x128"][1] == 1289756928
