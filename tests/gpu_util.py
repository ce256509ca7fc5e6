"""Thin torch-tensor wrappers over the C ABI for the GPU parity tests."""
import ctypes as C

import torch

from femasr_b200 import lib as L


def S():
    return torch.cuda.current_stream().cuda_stream


def p(t):
    return None if t is None else t.data_ptr()


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def nchw(x_nhwc):
    return x_nhwc.permute(0, 3, 1, 2).contiguous()


def pack_weight(w_oihw):
    lib = L.load()
    co, ci, kh, kw = w_oihw.shape
    out = torch.empty(kh * kw * ci, co, device=w_oihw.device)
    L.check(lib.femasr_pack_weight(p(w_oihw.contiguous()), p(out), co, ci, kh, kw, S()))
    return out


def igemm(x, w_packed, bias, B, Hin, Win, Cin, Cout, ksize=3, stride=1, upsample=0, prologue=0, pro_a=None,
          pro_b=None, gamma=None, beta=None, act=0, res1=None, res2=None, fn="femasr_igemm_simt", y=None):
    lib = L.load()
    He, We = (2 * Hin, 2 * Win) if upsample else (Hin, Win)
    if ksize == 1:
        Ho, Wo = Hin, Win
    elif stride == 1:
        Ho, Wo = He, We
    else:
        Ho, Wo = (He - 1) // 2 + 1, (We - 1) // 2 + 1
    if y is None:
        y = torch.empty(B, Ho, Wo, Cout, device=x.device)
    a = L.IgemmArgs(p(x), p(w_packed), p(bias), p(res1), p(res2), p(y), p(pro_a), p(pro_b), p(gamma), p(beta),
                    B, Hin, Win, Cin, Cout, ksize, stride, upsample, prologue, act)
    L.check(getattr(lib, fn)(C.byref(a), S()))
    return y


def gn_tables(x_nhwc, gamma, beta, eps=1e-6):
    lib = L.load()
    B, H, W, Cc = x_nhwc.shape
    sc = torch.empty(B, Cc, device=x_nhwc.device)
    sh = torch.empty(B, Cc, device=x_nhwc.device)
    scratch = torch.empty(max(1, lib.femasr_gn_scratch_floats(B, H * W, Cc)), device=x_nhwc.device)
    L.check(lib.femasr_gn_stats(p(x_nhwc), p(gamma), p(beta), p(sc), p(sh), p(scratch), B, H * W, Cc, eps, S()))
    return sc, sh


def ln_stats(x_tokens, eps=1e-5):
    lib = L.load()
    M, Cc = x_tokens.shape
    mu = torch.empty(M, device=x_tokens.device)
    rs = torch.empty(M, device=x_tokens.device)
    L.check(lib.femasr_ln_stats(p(x_tokens), p(mu), p(rs), M, Cc, eps, S()))
    return mu, rs


def tc_pack(w_oihw):
    lib = L.load()
    co, ci, kh, kw = w_oihw.shape
    blob = torch.empty(lib.femasr_tc_weight_bytes(co, ci, kh, kw), dtype=torch.uint8, device=w_oihw.device)
    w = w_oihw.contiguous()
    L.check(lib.femasr_tc_pack_weight(p(w), p(blob), co, ci, kh, kw, S()))
    return blob


def tc_prepare(x_nhwc, mode=0, pro_a=None, pro_b=None, gamma=None, beta=None, upsample=0, eps=1e-6):
    lib = L.load()
    B, H, W, Cc = x_nhwc.shape
    u = 2 if upsample else 1
    hi = torch.empty(B, H * u, W * u, Cc, dtype=torch.float16, device=x_nhwc.device)
    lo = torch.empty_like(hi)
    L.check(lib.femasr_tc_prepare(p(x_nhwc), p(hi), p(lo), mode, p(pro_a), p(pro_b), p(gamma), p(beta), B, H, W, Cc,
                                  upsample, eps, S()))
    return hi, lo


def tc_pack_f8(w_oihw, up2=False):
    """F8 cross-term packing of a conv weight (second plane: interleaved e4m3 bytes); up2: the sub-pixel phase filters."""
    lib = L.load()
    co, ci, kh, kw = w_oihw.shape
    w = w_oihw.contiguous()
    if up2:
        blob = torch.empty(lib.femasr_tc_weight_bytes(4 * co, ci, 2, 2), dtype=torch.uint8, device=w.device)
        L.check(lib.femasr_tc_pack_weight_up2_f8(p(w), p(blob), co, ci, S()))
    else:
        blob = torch.empty(lib.femasr_tc_weight_bytes(co, ci, kh, kw), dtype=torch.uint8, device=w.device)
        L.check(lib.femasr_tc_pack_weight_f8(p(w), p(blob), co, ci, kh, kw, S()))
    return blob


def tc_prepare_f8(x_nhwc, mode=0, pro_a=None, pro_b=None):
    """fp16 hi plane + the interleaved e4m3 plane (same byte size as a lo plane) of the F8 cross-term mode."""
    lib = L.load()
    B, H, W, Cc = x_nhwc.shape
    hi = torch.empty(B, H, W, Cc, dtype=torch.float16, device=x_nhwc.device)
    x8 = torch.empty(B, H, W, Cc, dtype=torch.float16, device=x_nhwc.device)      # raw bytes
    L.check(lib.femasr_tc_prepare_f8(p(x_nhwc), p(hi), p(x8), mode, p(pro_a), p(pro_b), B, H, W, Cc, S()))
    return hi, x8


def tc_pack_up2(w_oihw):
    lib = L.load()
    co, ci, _, _ = w_oihw.shape
    blob = torch.empty(lib.femasr_tc_weight_bytes(4 * co, ci, 2, 2), dtype=torch.uint8, device=w_oihw.device)
    w = w_oihw.contiguous()
    L.check(lib.femasr_tc_pack_weight_up2(p(w), p(blob), co, ci, S()))
    return blob


def tc_igemm(hi, lo, blob, bias, Cout, ksize=3, act=0, res1=None, res2=None, y=None, upsample=0, split_out=False,
             gn_partial=None, stride=1, kb_begin=0, kb_count=0, slice_kb=0, pair=-1, strip=-1, f8=0, out_planes=None):
    """out_planes: the caller's (hi, lo) output planes (implies split_out); y: the caller's fp32 output."""
    lib = L.load()
    B, H, W, Cin = hi.shape
    u = 2 if upsample else 1
    Ho, Wo = ((H + 2 - ksize) // 2 + 1, (W + 2 - ksize) // 2 + 1) if stride == 2 else (H * u, W * u)
    oh = ol = None
    if out_planes is not None:
        (oh, ol), split_out = out_planes, True
    elif split_out:
        oh = torch.empty(B, Ho, Wo, Cout, dtype=torch.float16, device=hi.device)
        ol = torch.empty_like(oh)
    elif y is None:
        y = torch.empty(B, Ho, Wo, Cout, device=hi.device)
    a = L.TcArgs(p(hi), p(lo), p(blob), p(bias), p(res1), p(res2), p(y), B, H, W, Cin, Cout, ksize, act,
                 p(oh), p(ol), stride, kb_begin, kb_count, slice_kb, pair, strip, p(gn_partial), upsample, f8)
    L.check(lib.femasr_tc_igemm(C.byref(a), S()))
    return (oh, ol) if split_out else y


def tc_gn_rows(B, H, W, Cin, Cout, upsample=0, stride=1, slice_kb=0, pair=-1, strip=-1):
    a = L.TcArgs(None, None, None, None, None, None, None, B, H, W, Cin, Cout, 3, 0, None, None, stride, 0, 0,
                 slice_kb, pair, strip, None, upsample)
    return L.load().femasr_tc_gn_partial_rows(C.byref(a))
