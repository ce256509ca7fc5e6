"""GPU: the VQ stage (femasr_vq_match_tc + femasr_vq_finish, femasr_vq_select, femasr_codebook_gather) against the formula
DESIGN.md section 5 says it implements, at the engine's codebooks, at row counts that give a CTA several m-tiles, and at
feature scales from 2^6 down to 2^-14.

The contract, stated once (`contract`):
  * A_r and B_j are the library's own femasr_row_sumsq (checked separately against fp64, next to ATen fp32's error);
  * C_rj is the fp64 dot product rounded once to fp32 (fp32 products are exact in fp64);
  * d_rj = fl(fl(A_r + B_j) - 2 C_rj) in separate fp32 operations, argmin with the lowest index on ties.
A row is set aside as ambiguous when a code that could decide it has an fp64 C within e_dim * 2^-52 * sum|z_k e_k| of an
fp32 rounding midpoint (two fp64 summation orders may round it differently); the count is printed (a few rows in a
hundred thousand: the bound is a worst case).
The bar is zero index mismatches.  ATen's own formula (oracle.vq_dist) is compared for the report only: each of its
disagreements must be a tie under ATen's arithmetic (within 2 of its grid steps).

Each fused case also checks the top-4 candidate list itself: ascending in (d, j), distinct valid codes, every candidate's
tensor-core distance within half the margin vq_finish_kernel computes for the row (restated in `finish_margin`), and the
exact argmin among the candidates the kernel refines, or the row rescanned."""
import math

import pytest
import torch

from femasr_b200 import lib as L
from femasr_b200.spec import random_state_dict
from oracle import femasr_oracle as O
from tests import gpu_util as G
from tests.test_engine_plan import CONFIGS

pytestmark = pytest.mark.gpu

NONE = 0x7fffffff                  # the code of an empty candidate slot
EPS32 = 2.0 ** -23


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (n_e, e_dim): every codebook of CONFIGS, plus BN = 64 code tiles (n_e not a multiple of 128) with one, three and five tiles
CODEBOOKS = sorted({(n, e) for _s, cbs, _sem, _tap in CONFIGS.values() for _cs, n, e in cbs}) + [(64, 64), (192, 64), (320, 128)]
assert {(1024, 256), (1024, 512), (512, 128), (512, 256), (256, 128)} <= set(CODEBOOKS)
ROWS = ("1", "127", "128", "129", "S128", "S128+1", "5S128+37")
SCALES = (6, 3, 0, -4, -8, -10, -12, -14)


def rows_of(name):
    S = sms()
    return {"1": 1, "127": 127, "128": 128, "129": 129, "S128": S * 128, "S128+1": S * 128 + 1,
            "5S128+37": 5 * S * 128 + 37, "131072": 131072}[name]


def make_case(n_e, e_dim, N, kind, k, seed):
    """z [N, e_dim] of std 2^k and a codebook: tiny = the reference's init U(+-1/n_e) (tie-heavy, kept at its init),
    randn = N(0, 1), trained = codes of std 2^k with every z row next to one of them (d << A)."""
    g = torch.Generator().manual_seed(seed)
    s = 2.0 ** k
    if kind == "tiny":
        cb = (torch.rand(n_e, e_dim, generator=g) * 2 - 1) / n_e
    else:
        cb = torch.randn(n_e, e_dim, generator=g) * (s if kind == "trained" else 1.0)
    if kind == "trained":
        z = cb[torch.randint(0, n_e, (N,), generator=g)] + 0.05 * s * torch.randn(N, e_dim, generator=g)
    else:
        z = torch.randn(N, e_dim, generator=g) * s
    return z, cb


# ------------------------------------------------------------------------------------------------ library calls
def row_sumsq(x):
    out = torch.empty(x.shape[0], device=x.device)
    L.check(L.load().femasr_row_sumsq(x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], G.S()))
    return out


def fused(z, cb):
    """femasr_vq_match_tc + femasr_vq_finish as the engine runs them; device tensors in, device tensors out."""
    lib = L.load()
    N, e_dim = z.shape
    n_e = cb.shape[0]
    a, b = row_sumsq(z), row_sumsq(cb)
    hi, lo = G.tc_prepare(z.view(1, 1, N, e_dim))
    blob = G.tc_pack(cb.view(n_e, e_dim, 1, 1))
    cand = torch.empty(N, 4, 2, dtype=torch.int32, device=z.device)
    L.check(lib.femasr_vq_match_tc(hi.data_ptr(), lo.data_ptr(), blob.data_ptr(), a.data_ptr(), b.data_ptr(),
                                   cand.data_ptr(), N, n_e, e_dim, G.S()))
    idx = torch.empty(N, dtype=torch.int64, device=z.device)
    zq = torch.empty(N, e_dim, device=z.device)
    lrows = torch.empty(N, device=z.device)
    st = torch.zeros(3, dtype=torch.int32, device=z.device)
    L.check(lib.femasr_vq_finish(z.data_ptr(), a.data_ptr(), cand.data_ptr(), cb.data_ptr(), b.data_ptr(), idx.data_ptr(),
                                 zq.data_ptr(), lrows.data_ptr(), st.data_ptr(), N, n_e, e_dim, G.S()))
    torch.cuda.synchronize()
    return dict(a=a, b=b, cand=cand, idx=idx, zq=zq, lrows=lrows, stats=st.tolist())


# ------------------------------------------------------------------------------------------------ the reference
def ulp_of(x):
    """Spacing of fp32 numbers at |x| (normal range), as vq.cu's ulp_of."""
    return (x.float().view(torch.int32) & 0x7f800000).view(torch.float32) * EPS32


def contract(z, cb, a, b, ours=None, cand_j=None, want_c=False, chunk=8192):
    """The contract argmin of every row, the ambiguous-row mask, and optionally: the contract distance of the candidate
    codes cand_j [N, 4] (inf for empty slots), the fp32 C matrix, and ATen's disagreements with `ours` as
    (row, grid gap) pairs.  Everything on the device, in row chunks."""
    N, e_dim = z.shape
    cb64 = cb.double()
    cbabs = cb64.abs().t()
    out = dict(idx=torch.empty(N, dtype=torch.int64, device=z.device),
               amb=torch.empty(N, dtype=torch.bool, device=z.device), aten=[])
    if cand_j is not None:
        out["dcand"] = torch.full((N, 4), math.inf, device=z.device)
    if want_c:
        out["c"] = torch.empty(N, cb.shape[0], device=z.device)
    b_aten = torch.sum(cb ** 2, 1)
    for r0 in range(0, N, chunk):
        r1 = min(N, r0 + chunk)
        zz = z[r0:r1].double()
        c64 = zz @ cb64.t()
        c = c64.float()
        ab = a[r0:r1, None] + b[None, :]
        d = ab - 2 * c
        i = torch.argmin(d, 1)                                  # first (lowest) index on ties
        out["idx"][r0:r1] = i
        # codes whose fp64 C may round the other way under another summation order
        tol = e_dim * 2.0 ** -52 * (zz.abs() @ cbabs)
        cd = c.double()
        up = torch.nextafter(c, torch.tensor(math.inf, device=z.device)).double()
        dn = torch.nextafter(c, torch.tensor(-math.inf, device=z.device)).double()
        near = torch.minimum((c64 - (cd + up) / 2).abs(), (c64 - (cd + dn) / 2).abs()) <= tol
        alt = torch.where(c64 >= cd, up, dn).float()
        # ... and could decide the row: the argmin rounded the other way reaching the runner-up, or another code reaching the best
        d12 = torch.topk(d, min(2, d.shape[1]), 1, largest=False).values
        dalt = ab - 2 * alt
        best = torch.arange(d.shape[1], device=z.device)[None, :] == i[:, None]
        out["amb"][r0:r1] = (near & torch.where(best, dalt >= d12[:, -1:], dalt <= d12[:, :1])).any(1)
        if cand_j is not None:
            cj = cand_j[r0:r1].long()
            ok = (cj >= 0) & (cj < cb.shape[0])
            out["dcand"][r0:r1] = torch.where(ok, d.gather(1, cj.clamp(0, cb.shape[0] - 1)), math.inf)
        if want_c:
            out["c"][r0:r1] = c
        if ours is not None:
            da = O.vq_dist(z[r0:r1], cb)                        # ATen's formula and summation order
            theirs = torch.argmin(da, 1)
            rows = torch.nonzero(ours[r0:r1] != theirs).reshape(-1)
            if rows.numel():
                o, t = ours[r0:r1][rows], theirs[rows]
                a_aten = torch.sum(z[r0:r1][rows] ** 2, 1)
                grid = ulp_of(torch.maximum((a_aten + b_aten[o]).abs(), (a_aten + b_aten[t]).abs()))
                gap = (da[rows, o] - da[rows, t]) / grid
                out["aten"] += list(zip((rows + r0).tolist(), gap.tolist()))
        del c64, c, ab, d, tol, cd, up, dn, near, alt
    return out


def finish_margin(a, b, cand_d, cand_j, e_dim):
    """vq_finish_kernel's margin per row (vq.cu): 2.5 ulps of max(|A + B_best|, |d_best|), plus the relative bound
    4 * eps * (3 e_dim / 16) * |A + B_best - d_best| and the absolute bound 2^-23 * sqrt(e_dim * max B of the candidates)."""
    j0 = cand_j[:, 0].long().clamp(0, b.numel() - 1)
    ab0 = a + b[j0]
    valid = cand_j != NONE
    bmax = torch.where(valid, b[cand_j.long().clamp(0, b.numel() - 1)], 0.0).amax(1)
    return (2.5 * ulp_of(torch.maximum(ab0.abs(), cand_d[:, 0].abs())) + 4 * EPS32 * (3 * e_dim // 16) * (ab0 - cand_d[:, 0]).abs()
            + 2.0 ** -23 * torch.sqrt(e_dim * bmax) + 1e-30)


def check_sums(z, a, what):
    """A (or B) of femasr_row_sumsq against fp64, next to ATen fp32 on the same rows; returns the two relative errors."""
    want = (z.double() ** 2).sum(1)
    den = want.clamp_min(1e-300)
    ours = ((a.double() - want).abs() / den).max().item()
    aten = (((z ** 2).sum(1).double() - want).abs() / den).max().item()
    assert ours <= 4 * aten + 2 * EPS32, f"{what}: row_sumsq relative error {ours:.2e} (ATen fp32 {aten:.2e})"
    return ours, aten


def check_fused(z, cb, res, label, aten_ties=True):
    """Every per-case check of the fused path; returns the largest candidate-error-to-half-margin ratio.  aten_ties=False:
    ATen's disagreements are printed only (where its own fp32 GEMM error spans more than 2 grid steps)."""
    N, e_dim = z.shape
    n_e = cb.shape[0]
    ea, aa = check_sums(z, res["a"], "A")
    eb, ab_ = check_sums(cb, res["b"], "B")
    cd = res["cand"][:, :, 0].contiguous().view(torch.float32)
    cj = res["cand"][:, :, 1]
    ref = contract(z, cb, res["a"], res["b"], ours=res["idx"], cand_j=cj)
    keep = ~ref["amb"]
    mism = int(((res["idx"] != ref["idx"]) & keep).sum())
    gaps = [round(g, 2) for _r, g in ref["aten"]]
    st = res["stats"]
    # candidate list: distinct valid codes, ascending in (d, j)
    assert bool(((cj >= 0) & (cj < n_e)).all()), f"{label}: candidate code out of range"
    assert bool((cj[:, :, None] != cj[:, None, :]).sum((1, 2)).eq(12).all()), f"{label}: repeated candidate"
    asc = (cd[:, 1:] > cd[:, :-1]) | ((cd[:, 1:] == cd[:, :-1]) & (cj[:, 1:] > cj[:, :-1]))
    assert bool(asc.all()), f"{label}: candidates not ascending in (d, j)"
    # each tensor-core distance within half the margin of its exact distance; the argmin among the refined candidates
    m = finish_margin(res["a"], res["b"], cd, cj, e_dim)
    ratio = ((cd - ref["dcand"]).abs() / (m[:, None] / 2)).max().item()
    nc = 1 + ((cd[:, 1:] - cd[:, :1]) <= m[:, None]).sum(1)
    inside = ((cj == ref["idx"][:, None]) & (torch.arange(4, device=cj.device)[None, :] < nc[:, None])).any(1)
    missed = int((~inside & (nc < 4) & keep).sum())
    print(f"{label}: mismatches {mism}/{N} (ambiguous {int(ref['amb'].sum())}), refined {st[0]}, rescanned {st[1]}, "
          f"changed {st[2]}, cand err / half margin {ratio:.3f}, ATen disagreements {len(gaps)} gaps {gaps[:8]}, "
          f"A err {ea:.1e} (ATen {aa:.1e}), B err {eb:.1e} (ATen {ab_:.1e})")
    assert mism == 0, f"{label}: {mism}/{N} index mismatches against the contract"
    assert ratio <= 1.0, f"{label}: a candidate's tensor-core distance is {ratio:.3f} half-margins from its exact distance"
    assert missed == 0, f"{label}: {missed} rows whose argmin is outside the refined candidates and were not rescanned"
    assert st[1] <= st[0] <= N
    assert not aten_ties or all(0.0 <= g <= 2.0 for g in gaps), f"{label}: an ATen disagreement is not a tie in its own arithmetic: {gaps}"
    # straight-through output, loss rows, loss sum
    e = cb[res["idx"]]
    assert torch.equal(res["zq"], z + (e - z)), f"{label}: zq is not z + (e - z) bit for bit"
    want_rows = ((e.double() - z.double()) ** 2).sum(1)
    assert torch.allclose(res["lrows"].double(), want_rows, rtol=2e-6, atol=0), f"{label}: loss rows"
    tot = torch.empty((), device=z.device)
    L.check(L.load().femasr_sum_scaled(res["lrows"].data_ptr(), tot.data_ptr(), N, 1.0 / (N * e_dim), G.S()))
    want_tot = res["lrows"].double().sum().item() / (N * e_dim)
    assert abs(tot.item() - want_tot) <= 2 * EPS32 * abs(want_tot), f"{label}: femasr_sum_scaled"
    return ratio


# ------------------------------------------------------------------------------------------------ case table
# every codebook at every row count (tie-heavy init, scale 1); three codebooks at every kind and scale (one multi-tile
# row count); 131072 rows (config 2 at batch 32) for the engine's main codebook at two scales
TABLE = ([pytest.param(n, e, r, "tiny", 0, id=f"{n}x{e}-N{r}-tiny-k0") for n, e in CODEBOOKS for r in ROWS] +
         [pytest.param(n, e, "S128+1", kind, k, id=f"{n}x{e}-NS128+1-{kind}-k{k}")
          for n, e in ((1024, 256), (512, 128), (192, 64)) for kind in ("tiny", "randn", "trained") for k in SCALES
          if not (kind == "tiny" and k == 0)] +
         [pytest.param(1024, 256, "131072", kind, k, id=f"1024x256-N131072-{kind}-k{k}")
          for kind, k in (("tiny", 0), ("tiny", -12), ("trained", -12))])


@pytest.mark.parametrize("n_e,e_dim,rows,kind,k", TABLE)
def test_vq_matrix(cuda, n_e, e_dim, rows, kind, k):
    N = rows_of(rows)
    z, cb = make_case(n_e, e_dim, N, kind, k, seed=1000 + n_e + e_dim + abs(k))
    z, cb = z.to(cuda), cb.to(cuda)
    check_fused(z, cb, fused(z, cb), f"{n_e}x{e_dim} N={N} {kind} 2^{k}")


@pytest.mark.parametrize("n_e,e_dim,rows,kind,k", [p for p in TABLE if p.values[2] != "131072"])
def test_vq_select_matrix(cuda, n_e, e_dim, rows, kind, k):
    """femasr_vq_select (gemm_path 0, FEMASR_VQ_FUSED=0) given the contract's C: exact."""
    N = rows_of(rows)
    z, cb = make_case(n_e, e_dim, N, kind, k, seed=1000 + n_e + e_dim + abs(k))
    z, cb = z.to(cuda), cb.to(cuda)
    a, b = row_sumsq(z), row_sumsq(cb)
    ref = contract(z, cb, a, b, want_c=True)
    idx = torch.empty(N, dtype=torch.int64, device=cuda)
    zq = torch.empty(N, e_dim, device=cuda)
    lrows = torch.empty(N, device=cuda)
    L.check(L.load().femasr_vq_select(z.data_ptr(), ref["c"].data_ptr(), cb.data_ptr(), b.data_ptr(), idx.data_ptr(),
                                      zq.data_ptr(), lrows.data_ptr(), N, n_e, e_dim, 0, G.S()))
    torch.cuda.synchronize()
    mism = int((idx != ref["idx"]).sum())
    assert mism == 0, f"{mism}/{N} index mismatches given the contract's C"
    e = cb[idx]
    assert torch.equal(zq, z + (e - z))
    assert torch.allclose(lrows.double(), ((e.double() - z.double()) ** 2).sum(1), rtol=2e-6, atol=0)


# exact duplicates of the best code where the top-4 merge sees them: columns 8j + 2q + e of one thread's fragment
STEPS = {"same-thread": 8, "same-lane": 1, "quad-lanes": 2, "code-tiles": None}     # None: one code tile (BN)
DUPS = [pytest.param(n, e, s, c, id=f"{n}x{e}-{s}-{c}") for n, e in ((1024, 256), (320, 128), (192, 64))
        for s in STEPS for c in (2, 3, 4, 5, 9)]


@pytest.mark.parametrize("n_e,e_dim,step,copies", DUPS)
def test_vq_duplicates(cuda, n_e, e_dim, step, copies):
    bn = 128 if n_e % 128 == 0 else 64
    st_ = STEPS[step] or bn
    c0 = 6                                                   # even: c0 and c0 + 1 are e = 0 and e = 1 of one lane
    pos = [c0 + st_ * i for i in range(copies)]
    if pos[-1] >= n_e:
        pytest.skip(f"{copies} copies {st_} apart do not fit in {n_e} codes")
    g = torch.Generator().manual_seed(77 + copies)
    cb = torch.randn(n_e, e_dim, generator=g)
    for p_ in pos[1:]:
        cb[p_] = cb[c0]
    N = 257
    z = cb[c0] + 1e-3 * torch.randn(N, e_dim, generator=g)
    z, cb = z.to(cuda), cb.to(cuda)
    res = fused(z, cb)
    check_fused(z, cb, res, f"{n_e}x{e_dim} {copies} copies {st_} apart")
    assert bool((res["idx"] == c0).all()), "a duplicate with a higher index won"
    top = min(copies, 4)                                     # equal distances: the list holds the lowest-index copies
    assert res["cand"][:, :top, 1].eq(torch.tensor(pos[:top], device=cuda)).all(), "top-4 merge lost a lower-index copy"
    st = res["stats"]
    assert st[0] == N and st[1] == (N if copies >= 4 else 0), f"refined / rescanned {st[:2]}"


@pytest.mark.parametrize("k", [-12, -10])
def test_vq_equidistant_codes(cuda, k):
    """Eight feature rows of std 2^k, each with nine codes at the same exact distance in orthogonal directions: their fp32
    distances differ by a few grid steps while the tensor-core error of small z spreads them by ~100, so the exact argmin
    is often not in the tensor-core top 4.  All nine lie inside the margin, so these rows must be rescanned.  ATen's fp32
    GEMM spreads them just as much, so its disagreements here are reported, not bounded."""
    n_e, e_dim, reps = 1024, 256, 16
    g = torch.Generator().manual_seed(94)
    cb = (torch.rand(n_e, e_dim, generator=g) * 2 - 1) / n_e
    centres = torch.randn(8, e_dim, generator=g) * 2.0 ** k
    for c in range(8):
        q = torch.linalg.qr(torch.randn(e_dim, 9, generator=g, dtype=torch.float64))[0].t()
        for i in range(9):
            cb[100 * c + 8 * i + 6] = (centres[c].double() + 3e-3 * q[i]).float()
    z = centres.repeat_interleave(reps, 0)
    z, cb = z.to(cuda), cb.to(cuda)
    res = fused(z, cb)
    check_fused(z, cb, res, f"equidistant 2^{k}", aten_ties=False)
    assert res["stats"][1] == z.shape[0], f"rescanned {res['stats'][1]} of {z.shape[0]} rows"


@pytest.mark.parametrize("kind,k", [("tiny", 0), ("tiny", -12), ("trained", -8)])
def test_vq_batch_invariance(cuda, kind, k):
    """Rows of a 5 S 128 + 37 batch (several m-tiles per CTA) equal the same rows run as a 129-row batch, bit for bit in
    cand, idx and zq; a second run is bit-identical."""
    n_e, e_dim = 1024, 256
    N = rows_of("5S128+37")
    z, cb = make_case(n_e, e_dim, N, kind, k, seed=91)
    z, cb = z.to(cuda), cb.to(cuda)
    big, again = fused(z, cb), fused(z, cb)
    for key in ("cand", "idx", "zq", "lrows"):
        assert torch.equal(big[key], again[key]), f"second run differs in {key}"
    for r0 in (3 * sms() * 128 - 64, N - 129):
        part = fused(z[r0:r0 + 129].contiguous(), cb)
        for key in ("cand", "idx", "zq"):
            assert torch.equal(part[key], big[key][r0:r0 + 129]), f"rows {r0}..: {key} depends on the batch"


def test_vq_nan_row(cuda):
    """A z row holding NaN gets index 0 (as torch.argmin of an all-NaN row) and leaves every other row unchanged."""
    n_e, e_dim = 1024, 256
    N = rows_of("S128+1")
    z, cb = make_case(n_e, e_dim, N, "tiny", 0, seed=92)
    z, cb = z.to(cuda), cb.to(cuda)
    clean = fused(z, cb)
    bad = [0, 200, N - 1]
    zn = z.clone()
    zn[bad, 3] = math.nan
    res = fused(zn, cb)
    assert bool((res["idx"][bad] == 0).all()), f"NaN rows got {res['idx'][bad].tolist()}"
    other = torch.ones(N, dtype=torch.bool, device=cuda)
    other[bad] = False
    for key in ("cand", "idx", "zq", "lrows"):
        assert torch.equal(res[key][other], clean[key][other]), f"a NaN row changed {key} of other rows"


@pytest.mark.parametrize("n_e,e_dim", CODEBOOKS)
def test_codebook_gather(cuda, n_e, e_dim):
    """femasr_codebook_gather (decode_indices) equals cb[idx] bit for bit."""
    N = rows_of("5S128+37")
    g = torch.Generator().manual_seed(93)
    cb = torch.randn(n_e, e_dim, generator=g).to(cuda)
    idx = torch.randint(0, n_e, (N,), generator=g).to(cuda)
    idx[:3] = torch.tensor([0, n_e - 1, n_e - 1])
    zq = torch.empty(N, e_dim, device=cuda)
    L.check(L.load().femasr_codebook_gather(idx.data_ptr(), cb.data_ptr(), zq.data_ptr(), N, n_e, e_dim, G.S()))
    torch.cuda.synchronize()
    assert torch.equal(zq, cb[idx])


# ------------------------------------------------------------------------------------------------ engine level
def engine_rows(cuda, scale, cbs, B, H, gemm_path, seed):
    from basicsr.archs.femasr_arch import FeMaSRNet
    sd = random_state_dict(scale, cbs[0][2], seed=seed, init="default", codebooks=cbs if len(cbs) > 1 else None)
    net = FeMaSRNet(codebook_params=cbs, LQ_stage=True, scale_factor=scale, gemm_path=gemm_path)
    net.load_state_dict(sd, strict=True)
    net = net.to(cuda).eval()
    x = torch.rand(B, 3, H, H, generator=torch.Generator().manual_seed(1))
    names = ["z", "z1", "z2"][:len(cbs)]
    _out, _loss, idx, taps = net._native(cuda).forward(x.to(cuda), taps=names)
    idx = idx if isinstance(idx, list) else [idx]
    res = []
    for k, name in enumerate(names):
        cb = sd[f"quantize_group.{k}.embedding.weight"].to(cuda)
        z = taps[name].reshape(-1, cb.shape[1])
        res.append((name, z, cb, idx[k].reshape(-1)))
    return res


def engine_check(z, cb, ours, label, bound=True):
    ref = contract(z, cb, row_sumsq(z), row_sumsq(cb), ours=ours)
    keep = ~ref["amb"]
    mism = int(((ours != ref["idx"]) & keep).sum())
    gaps = [round(g, 2) for _r, g in ref["aten"]]
    print(f"{label}: {mism}/{z.shape[0]} mismatches against the contract (ambiguous {int(ref['amb'].sum())}), "
          f"z std {z.std().item():.3g}, ATen disagreements {len(gaps)} gaps {gaps[:16]}")
    if bound:
        assert mism == 0, f"{label}: {mism} index mismatches"
        assert all(0.0 <= g <= 2.0 for g in gaps), f"{label}: an ATen disagreement is not a tie: {gaps}"


def test_engine_config2_full_batch(cuda):
    """Config 2 at batch 32 (131072 rows, about 8 m-tiles per CTA) on the tensor-core path: 0 mismatches; the fp32 FFMA
    path (gemm_path 0, no refinement) is reported only."""
    for gemm_path in (1, 0):
        for name, z, cb, ours in engine_rows(cuda, 4, [[32, 1024, 256]], 32, 128, gemm_path, seed=0):
            engine_check(z, cb, ours, f"config 2 b32 gemm_path {gemm_path} {name}", bound=gemm_path == 1)
            if gemm_path == 1:
                res = fused(z, cb)              # the same stage outside the engine, with its refinement counters
                st = res["stats"]
                print(f"config 2 b32: refined {st[0]} ({st[0] / z.shape[0]:.2%}), rescanned {st[1]}, changed {st[2]}")
                assert torch.equal(res["idx"], ours)


def test_engine_x2_cb3(cuda):
    """x2_cb3 (three codebooks: 1024 x 512, 512 x 256, 256 x 128) at a small batch, every level's tap."""
    scale, cbs, _sem, _tap = CONFIGS["x2_cb3"]
    for name, z, cb, ours in engine_rows(cuda, scale, cbs, 2, 128, 1, seed=3):
        engine_check(z, cb, ours, f"x2_cb3 {name} ({cb.shape[0]} x {cb.shape[1]})")
