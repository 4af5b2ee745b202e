"""CPU: the exact-operand sweep of test_gemm_exact_gpu.py against an emulation of the GEMM's index maps, and against broken variants.

``emulate_gemm`` / ``emulate_conv`` / ``emulate_wgrad`` restate where gemm_sm90.cu takes every value from: 128 x 256 tiles,
64-deep k-blocks, decode_unit's split ranges, TMA boxes zero-filled past the tensor (K-major 64 x 128 / 64 x 256, MN-major
64 x 64), GEGLU's 3-D map pairing 128 h rows with the same 128 gate rows, the convolution's 4-D box {64, W, hb, nb} shifted by
each tap, the weight gradient's per-box tap shift, t = bf16(fp32(acc) + bias) per column, the epilogue's 8-column chunks with
their n_ok < 8 tail, and the per-image aux row row / (H W).  On the sweep's exact operands the emulation must match the float64
reference bit for bit, and every mutant -- one local mistake of the kind a kernel change makes -- must change some bit of some
case of the sweep: that is what proves the sweep crosses each edge the mutant breaks."""
import pytest
import torch

import cflearn_b200  # noqa: F401  (registers the package)
from cflearn_b200 import ops
from _refs import EXACT_BUDGET, bf16, cancel_pairs, conv3x3_dgrad, exact_operands, gemm_epilogue, gemm_t, splitk_ranges
import test_gemm_exact_gpu as sweep

F64 = torch.float64
BM, BN, BK = 128, 256, 64
MUTANTS = ["last_partial_kblock_dropped", "split_boundary_off_by_one", "partial_tile_last_row_shifted", "tail_columns_dropped",
           "bias_of_next_column", "halo_wrapped", "ky_kx_transposed", "dgrad_taps_not_flipped", "aux_by_tile", "geglu_wrong_half",
           "round_half_away", "split_planes_swapped", "acc_bf16_between_kblocks", "acc_16_bits", "wgrad_tap_of_first_box"]


# ---- emulation ------------------------------------------------------------------------------------------------------------------------
def box(t, starts, sizes):
    """A TMA box of t (dims outermost first): t[s : s + n] along every dim, zero where that falls outside t."""
    out = torch.zeros(sizes, dtype=torch.float32)
    src, dst = [], []
    for s, n, d in zip(starts, sizes, t.shape):
        lo, hi = max(s, 0), min(s + n, d)
        if hi <= lo:
            return out
        src.append(slice(lo, hi))
        dst.append(slice(lo - s, hi - s))
    out[tuple(dst)] = t[tuple(src)].float()
    return out


def round_bf16(x, mutant):
    """fp32 -> bf16: round to nearest even, or (mutant) half away from zero."""
    if mutant != "round_half_away":
        return x.to(torch.bfloat16)
    bits = x.view(torch.int32).long() & 0xFFFFFFFF
    bits = ((bits + 0x8000) >> 16) & 0xFFFF
    return (bits - (bits >= 0x8000).long() * 0x10000).to(torch.int16).view(torch.bfloat16)


def accumulate(acc, a, b, last, mutant):
    """acc += a b^T over one k-block (exact in fp32 on the sweep's operands); the mutants narrow the accumulator between k-blocks."""
    acc = acc + a @ b.t()
    if not last and mutant == "acc_bf16_between_kblocks":
        acc = acc.to(torch.bfloat16).float()
    if not last and mutant == "acc_16_bits":  # keep 16 significant bits
        m, e = torch.frexp(acc)
        acc = torch.ldexp(torch.trunc(m * 2.0 ** 16) / 2.0 ** 16, e)
    return acc


def split_bounds(nkb, splits, mutant):
    s = min(splits, nkb)
    b = [nkb * sp // s for sp in range(s + 1)]
    if mutant == "split_boundary_off_by_one":
        b = [b[0]] + [min(v + 1, nkb) for v in b[1:-1]] + [b[-1]]
    return [(b[sp], b[sp + 1]) for sp in range(s)]


def mainloop(M, n_tiles, nkb, splits, load_a, load_b, mutant):
    """Yields (m tile, n tile, split, fp32 accumulator [128, 256]) of every work unit."""
    for m_t in range((M + BM - 1) // BM):
        for n_t in range(n_tiles):
            for sp, (kb0, kb1) in enumerate(split_bounds(nkb, splits, mutant)):
                acc = torch.zeros(BM, BN)
                for kb in range(kb0, kb1):
                    if mutant == "last_partial_kblock_dropped" and kb == nkb - 1 and load_a.partial_last:
                        continue
                    acc = accumulate(acc, load_a(m_t, kb), load_b(n_t, kb), kb == kb1 - 1, mutant)
                yield m_t, n_t, sp, acc


def store(T, m_t, cols, tile, mutant):
    """The epilogue's stores of one tile: rows below M, 8-column chunks of the output columns ``cols`` [256] (-1: none)."""
    M, width = T.shape
    rows = min(BM, M - m_t * BM)
    src = torch.arange(rows)
    if mutant == "partial_tile_last_row_shifted" and rows < BM:
        src[-1] += 1
    ok = (cols >= 0) & (cols < width)
    if mutant == "tail_columns_dropped":  # a chunk with n_ok < 8 writes nothing
        chunk_full = ok.view(-1, 8).all(1, keepdim=True).expand(-1, 8).reshape(-1)
        ok = ok & chunk_full
    T[m_t * BM: m_t * BM + rows, cols[ok]] = tile[src][:, ok]


def make_loaders(A_store, a_mn, B_store, b_mn, K, paired_F=None, mutant=None):
    """Box loaders of the A tile [128, 64] and the B tile [256, 64] of (tile, k-block), from the operands as stored."""
    def load_a(m_t, kb):
        if not a_mn:
            return box(A_store, (m_t * BM, kb * BK), (BM, BK))
        return torch.cat([box(A_store, (kb * BK, m_t * BM + i * 64), (BK, 64)).t() for i in range(BM // 64)])

    def load_b(n_t, kb):
        if paired_F is not None:  # W1 [2F, K] as {K, F, 2}: 128 h rows, then the same 128 rows of the gate half
            halves = B_store.view(2, paired_F, -1)
            g_t = n_t + 1 if mutant == "geglu_wrong_half" else n_t
            return torch.cat([box(halves[0], (n_t * 128, kb * BK), (128, BK)), box(halves[1], (g_t * 128, kb * BK), (128, BK))])
        if not b_mn:
            return box(B_store, (n_t * BN, kb * BK), (BN, BK))
        return torch.cat([box(B_store, (kb * BK, n_t * BN + i * 64), (BK, 64)).t() for i in range(BN // 64)])

    load_a.partial_last = K % BK != 0
    return load_a, load_b


def emulate_gemm(epi, a_mn, b_mn, A, B, bias, aux, splits, mutant=None):
    """The outputs of one b200_gemm_bf16 call (as gemm_epilogue gives them; the planes for EPI 4) on A [M, K], B [cols, K]."""
    M, K = A.shape
    cols = B.shape[0]
    N = 2 * cols if epi == 8 else cols
    nkb = (K + BK - 1) // BK
    paired = epi == 7
    load_a, load_b = make_loaders(A.t() if a_mn else A, a_mn, B.t() if b_mn else B, b_mn, K, N // 2 if paired else None, mutant)
    width = N // 2 if epi in (7, 8) else N  # the GEMM's own width
    n_tiles = (width + (128 if paired else BN) - 1) // (128 if paired else BN)
    s = min(splits, nkb)
    T = torch.full((s * M, N) if epi == 4 else (M, cols), float("nan"), dtype=torch.float32 if epi == 4 else torch.bfloat16)
    bias_pad = torch.zeros(N + BN + 1, dtype=F64)
    if bias is not None:
        bias_pad[:N] = bias.double()
    shift = 1 if mutant == "bias_of_next_column" else 0
    for m_t, n_t, sp, acc in mainloop(M, n_tiles, nkb, splits, load_a, load_b, mutant):
        c = torch.arange(BN)
        if paired:  # tile column c < 128: h column f = 128 n_t + c; c >= 128: the gate column F + f
            f = n_t * 128 + c % 128
            out_cols = torch.where(f < width, f + (c >= 128).long() * width, -1)
        else:
            out_cols = n_t * BN + c
        if epi == 4:
            tile = acc
            planes = T[sp * M:(sp + 1) * M]
            ok = out_cols < N
            rows = min(BM, M - m_t * BM)
            planes[m_t * BM: m_t * BM + rows, out_cols[ok]] = tile[:rows][:, ok]
            continue
        b = bias_pad[out_cols.clamp_min(0) + shift].float() if epi not in (3, 6, 8) else torch.zeros(BN)
        store(T, m_t, out_cols, round_bf16(acc + b, mutant), mutant)
    if epi == 4:
        if mutant == "split_planes_swapped" and s > 1:
            T = torch.cat([T[M:2 * M], T[:M], T[2 * M:]])
        return {"out0": T}
    return {k: v for k, (v, _) in gemm_epilogue(epi, T, aux).items()}


def emulate_conv(x, wp, bias, aux, epi, mutant=None):
    """The output of one b200_conv3x3_nhwc_bf16 call: x [B, H, W, Cin], w_packed [Cout, 9 Cin]."""
    Bn, H, W, Cin = x.shape
    Cout = wp.shape[0]
    M, HW, cpb = Bn * H * W, H * W, Cin // BK
    hb = min(H, BM // W)
    nb = BM // (W * hb)
    xf = x.reshape(M, Cin)

    def load_a(m_t, kb):
        tap, c0 = kb // cpb, (kb % cpb) * BK
        ky, kx = (tap % 3, tap // 3) if mutant == "ky_kx_transposed" else (tap // 3, tap % 3)
        m0 = m_t * BM
        if mutant == "halo_wrapped":  # the flat pixel sequence shifted: the halo wraps into the next row / image
            p = m0 + torch.arange(BM) + (ky - 1) * W + (kx - 1)
            ok = (p >= 0) & (p < M)
            out = torch.zeros(BM, BK)
            out[ok] = xf[p[ok], c0:c0 + BK].float()
            return out
        bimg = m0 // HW
        y0 = (m0 - bimg * HW) // W
        return box(x, (bimg, y0 + ky - 1, kx - 1, c0), (nb, hb, W, BK)).reshape(BM, BK)

    load_a.partial_last = False
    _, load_b = make_loaders(None, 0, wp, 0, 9 * Cin)
    T = torch.full((M, Cout), float("nan"), dtype=torch.bfloat16)
    bias_pad = torch.zeros(Cout + BN + 1, dtype=F64)
    if bias is not None:
        bias_pad[:Cout] = bias.double()
    shift = 1 if mutant == "bias_of_next_column" else 0
    n_tiles = (Cout + BN - 1) // BN
    for m_t, n_t, _, acc in mainloop(M, n_tiles, 9 * cpb, 1, load_a, load_b, mutant):
        cols = n_t * BN + torch.arange(BN)
        store(T, m_t, cols, round_bf16(acc + bias_pad[cols + shift].float(), mutant), mutant)
    aux_rows = aux
    if epi == 10:
        img = torch.arange(M) // HW
        if mutant == "aux_by_tile":
            img = torch.arange(M) // BM
        aux_rows = torch.full((M, Cout), float("nan"), dtype=aux.dtype)
        aux_rows[img < Bn] = aux[img[img < Bn]]
    return {k: v for k, (v, _) in gemm_epilogue(epi, T, aux_rows).items()}


def emulate_wgrad(x, dy, splits, mutant=None):
    """The planes [s Cout, 9 Cin] of one b200_conv3x3_wgrad_nhwc_bf16 call: x [B, H, W, Cin], dy [B H W, Cout]."""
    Bn, H, W, Cin = x.shape
    M, Cout = dy.shape
    HW, N = H * W, 9 * Cin
    xf = x.reshape(M, Cin)
    load_a, _ = make_loaders(dy, 1, None, 1, M)

    def load_b(n_t, kb):
        p0 = kb * BK
        bimg = p0 // HW
        y0 = (p0 - bimg * HW) // W
        parts = []
        for i in range(BN // 64):
            n = n_t * BN + i * 64
            tap, c0 = (n_t * BN if mutant == "wgrad_tap_of_first_box" else n) // Cin, n % Cin
            ky, kx = (tap % 3, tap // 3) if mutant == "ky_kx_transposed" else (tap // 3, tap % 3)
            if tap >= 9:
                parts.append(torch.zeros(64, BK))
            elif mutant == "halo_wrapped":
                p = p0 + torch.arange(BK) + (ky - 1) * W + (kx - 1)
                ok = (p >= 0) & (p < M)
                blk = torch.zeros(BK, 64)
                blk[ok] = xf[p[ok], c0:c0 + 64].float()
                parts.append(blk.t())
            else:
                parts.append(box(x, (bimg, y0 + ky - 1, kx - 1, c0), (1, BK // W, W, 64)).reshape(BK, 64).t())
        return torch.cat(parts)

    load_a.partial_last = False
    nkb = M // BK
    s = min(splits, nkb)
    T = torch.full((s * Cout, N), float("nan"))
    for m_t, n_t, sp, acc in mainloop(Cout, (N + BN - 1) // BN, nkb, splits, load_a, load_b, mutant):
        rows, cols = min(BM, Cout - m_t * BM), n_t * BN + torch.arange(BN)
        ok = cols < N
        T[sp * Cout + m_t * BM: sp * Cout + m_t * BM + rows, cols[ok]] = acc[:rows][:, ok]
    if mutant == "split_planes_swapped" and s > 1:
        T = torch.cat([T[Cout:2 * Cout], T[:Cout], T[2 * Cout:]])
    return {"out0": T}


# ---- the sweep, on the CPU ------------------------------------------------------------------------------------------------------------
def _same(got, want):
    """Bit-identical, NaN included."""
    bits = {torch.bfloat16: torch.int16, torch.float32: torch.int32, F64: torch.int64}
    return all(g.dtype == w.dtype and torch.equal(g.view(bits[g.dtype]), w.view(bits[w.dtype])) for g, w in
               ((got[k], want[k]) for k in want))


def gemm_sweep():
    """Every GEMM case of the GPU sweep: (name, epi, a_mn, b_mn, (A, B, bias, aux), splits, cancel)."""
    for epi, a_mn, b_mn in sweep.GEMM_EPIS:
        for i, (M, N, K, splits, cancel) in enumerate(sweep.gemm_cases(epi)):
            if splits == "pick":
                splits = ops.pick_splits(M, N, K)
            if M * N > 2 ** 22:
                continue  # the 136-tile case only checks grid independence; its single k-block is covered by smaller ones
            yield (f"gemm epi {epi} ({a_mn}, {b_mn}) {M}x{N}x{K} splits {splits} cancel {cancel}", epi, a_mn, b_mn,
                   sweep.gemm_inputs(epi, M, N, K, cancel, seed=1000 * epi + 10 * i, with_bias=i % 2 == 0), splits, cancel)


def gemm_case_results(mutant=None):
    """(name, emulation == reference) of every GEMM case; a mutant stops at its first rejection."""
    for name, epi, a_mn, b_mn, (A, B, bias, aux), splits, _ in gemm_sweep():
        want = {k: v for k, (v, _) in sweep.gemm_expected(epi, A, B, bias, aux, splits, device="cpu").items()}
        ok = _same(emulate_gemm(epi, a_mn, b_mn, A, B, bias, aux, splits, mutant), want)
        yield name, ok
        if mutant and not ok:
            return


def conv_case_results(mutant=None):
    for Bn, H, W, Cin, Cout, epi in sweep.CONV_CASES:
        x, w, bias, aux = sweep.conv_inputs(Bn, H, W, Cin, Cout, epi, seed=Bn * H * W + Cin + Cout + epi)
        want = {k: v for k, (v, _) in sweep.conv_expected(epi, x, w, bias, aux, device="cpu").items()}
        ok = _same(emulate_conv(x, ops.pack_conv3x3_weight(w), bias, aux, epi, mutant), want)
        yield f"conv epi {epi} {Bn}x{H}x{W}x{Cin}->{Cout}", ok
        if mutant and not ok:
            return
    for Bn, H, W, Cin, Cout in sweep.DGRAD_CASES:
        dy, w = sweep.dgrad_inputs(Bn, H, W, Cin, Cout)
        wp = ops.pack_conv3x3_weight(w.transpose(0, 1)) if mutant == "dgrad_taps_not_flipped" else ops.pack_conv3x3_weight_dgrad(w)
        ok = _same(emulate_conv(dy, wp, None, None, 0, mutant), {"out0": bf16(conv3x3_dgrad(dy, w))})
        yield f"dgrad {Bn}x{H}x{W}x{Cin}<-{Cout}", ok
        if mutant and not ok:
            return
    for Bn, H, W, Cin, Cout, splits in sweep.WGRAD_CASES:
        if splits == "pick":
            splits = ops.pick_splits(Cout, 9 * Cin, Bn * H * W)
        x, dy = sweep.wgrad_inputs(Bn, H, W, Cin, Cout)
        ok = _same(emulate_wgrad(x, dy, splits, mutant), {"out0": sweep.wgrad_planes(x, dy, splits).float()})
        yield f"wgrad {Bn}x{H}x{W}x{Cin}->{Cout} splits {splits}", ok
        if mutant and not ok:
            return


# ---- tests ----------------------------------------------------------------------------------------------------------------------------
def test_generator_is_exact_in_any_summation_order():
    """fp32 sums of the products -- forward, reverse and in k16 blocks -- equal the float64 value for every GEMM case of the sweep,
    and every case keeps sum |a b| under the budget (exact_operands asserts it)."""
    for name, epi, _, _, (A, B, _, _), _, cancel in gemm_sweep():
        K = A.shape[1]
        if cancel is not None:  # the cancelling pair is where the sweep says it is
            kp, kn = cancel_pairs(K, cancel)
            assert bool((A[:, kp] != 0).all() and (B[:, kp] == -B[:, kn]).all() and (A[:, kp] == A[:, kn]).all())
        exact = A.double() @ B.double().t()
        a, b = A.float(), B.float()
        fwd, rev, blk = (torch.zeros(A.shape[0], B.shape[0]) for _ in range(3))
        for k in range(K):
            fwd += a[:, k:k + 1] * b[:, k]
            rev += a[:, K - 1 - k:K - k] * b[:, K - 1 - k]
        for k0 in range(0, K, 16):
            part = torch.zeros_like(blk)
            for k in range(k0, min(K, k0 + 16)):
                part += a[:, k:k + 1] * b[:, k]
            blk += part
        for order, s in (("forward", fwd), ("reverse", rev), ("k16 blocks", blk)):
            assert torch.equal(s.double(), exact), f"{name}: fp32 sum in {order} order is not exact"


def test_budget_is_enforced():
    """Two cancelling pairs (4 x 2^20 units) break the 2^22 budget: the generator refuses them."""
    e = torch.zeros(4, dtype=F64)
    A, B = exact_operands(4, 4, 64, e, e, cancel=(0, 1))
    assert (A.double().abs() @ B.double().abs().t()).max() < EXACT_BUDGET
    with pytest.raises(AssertionError, match="budget"):
        exact_operands(4, 4, 64, e, e, cancel=(0, 1, 2, 3))


@pytest.mark.parametrize("family", ["gemm", "conv"])
def test_emulation_matches_the_reference_bit_for_bit(family):
    for name, ok in (gemm_case_results() if family == "gemm" else conv_case_results()):
        assert ok, f"{name}: the emulation differs from the float64 reference"


@pytest.mark.parametrize("mutant", MUTANTS)
def test_the_sweep_rejects_every_mutant(mutant):
    results = list(gemm_case_results(mutant)) + list(conv_case_results(mutant))
    assert not all(ok for _, ok in results), f"{mutant}: every case of the sweep still matches the reference bit for bit"


def test_rounding_and_split_ranges():
    x = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 1 + 2 ** -9, 1.5])
    assert round_bf16(x, None).tolist() == [1.0, 1 + 2 ** -6, -1.0, 1.0, 1.5]
    assert round_bf16(x, "round_half_away").tolist() == [1 + 2 ** -7, 1 + 2 ** -6, -(1 + 2 ** -7), 1.0, 1.5]
    assert torch.equal(gemm_t(torch.tensor([[257.0]], dtype=F64)).float(), torch.tensor([[256.0]]))
    assert splitk_ranges(65, 3) == [(0, 64), (64, 65)] and splitk_ranges(64 * 7, 3) == [(0, 128), (128, 256), (256, 448)]
