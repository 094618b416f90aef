"""Pins the CPU oracle (oracle/) before anything is compared against it.

Re-expresses, with fixed seeds, every property the reference's own tests
assert for this path (the reference has no golden vectors, SURVEY.md section 4):
  * quaternary scalar == digit dot        x86_64.rs:454-505
  * quaternary/binary/octal AVX2 == scalar x86_64.rs:544-602, 784-816
  * count_ones_simd == u32::count_ones     x86_64.rs:673-746
  * MetricResult ordering                  types.rs:1610-1633
and checks each formula against an independent restatement (numpy / exact
integer f32 emulation in tests/f32emu.py).
"""
import math
import struct

import numpy as np
import pytest

import oracle as orc
from oracle.pyoracle import lib, _p
from tests import f32emu


def rng(seed):
    return np.random.default_rng(seed)


# ------------------------------------------------------------------ synthetic

def test_synth_generator_is_counter_based_and_in_range():
    a = orc.synth(7, 0, 4096)
    b = orc.synth(7, 1000, 100)
    assert np.array_equal(a[1000:1100], b)
    assert a.min() >= -1.0 and a.max() < 1.0
    assert abs(float(a.mean())) < 0.05
    # python restatement of the documented formula
    M = (1 << 64) - 1

    def ref(seed, idx):
        z = (seed + idx * 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        z = z ^ (z >> 31)
        return ((z >> 40) - (1 << 23)) / float(1 << 23)

    for i in (0, 1, 17, 4095):
        assert a[i] == np.float32(ref(7, i))


# ----------------------------------------------------------------------- half

def test_f16_conversions_match_numpy_ieee_rne():
    r = rng(1)
    xs = np.concatenate([
        r.uniform(-1, 1, 2000).astype(np.float32),
        r.normal(0, 1e-4, 500).astype(np.float32),
        r.normal(0, 7e4, 300).astype(np.float32),       # overflow to inf
        np.array([0.0, -0.0, 1.0, -1.0, 65504.0, 65520.0, 65519.99, 5.96e-8, 2.98e-8, 2.9802322e-8,
                  6.1e-5, 6.097555e-5, np.inf, -np.inf], dtype=np.float32),
    ])
    got = orc.f32_to_f16_bits(xs)
    want = xs.astype(np.float16).view(np.uint16)
    assert np.array_equal(got, want)
    L = lib()
    allh = np.arange(0, 1 << 16, dtype=np.uint16)
    finite = ~np.isnan(allh.view(np.float16))
    back = np.array([L.orc_f16_to_f32(int(h)) for h in allh[finite]], dtype=np.float32)
    assert np.array_equal(back.view(np.uint32), allh[finite].view(np.float16).astype(np.float32).view(np.uint32))


# ---------------------------------------------------------------- dot products

@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 31, 32, 33, 128, 768, 1000, 1024])
def test_dot_f32_simd_matches_exact_fma_lane_model(n):
    r = rng(100 + n)
    a = r.uniform(-1, 1, n).astype(np.float32)
    b = r.uniform(-1, 1, n).astype(np.float32)
    got = orc.dot_f32_simd(a, b)
    want = np.float32(f32emu.dot_f32_simd_order(a, b))
    assert struct.pack("<f", got) == struct.pack("<f", want)


def test_dot_f32_scalar_and_mag_are_sequential_no_fma():
    r = rng(5)
    a = r.uniform(-1, 1, 257).astype(np.float32)
    b = r.uniform(-1, 1, 257).astype(np.float32)
    L = lib()
    got = np.float32(L.orc_dot_f32_scalar(_p(a), _p(b), a.size))
    s = 0.0
    for x, y in zip(a, b):
        s = f32emu.add32(s, f32emu.mul32(float(x), float(y)))
    assert got == np.float32(s)
    assert orc.mag_f32(a) == np.float32(math.sqrt(f32emu.sumsq_sequential(a))) or \
        orc.mag_f32(a) == np.sqrt(np.float32(f32emu.sumsq_sequential(a)))


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 64, 100, 768, 4096])
def test_dot_u8_avx2_equals_scalar_equals_numpy(n):
    r = rng(200 + n)
    a = r.integers(0, 256, n, dtype=np.uint8)
    b = r.integers(0, 256, n, dtype=np.uint8)
    L = lib()
    s = L.orc_dot_u8_scalar(_p(a), _p(b), n)
    v = L.orc_dot_u8_avx2(_p(a), _p(b), n)
    assert s == v == int((a.astype(np.uint64) * b.astype(np.uint64)).sum())


def test_dot_f16_is_sequential_f32():
    r = rng(6)
    a = r.uniform(-1, 1, 300).astype(np.float16)
    b = r.uniform(-1, 1, 300).astype(np.float16)
    L = lib()
    au, bu = a.view(np.uint16), b.view(np.uint16)
    got = np.float32(L.orc_dot_f16(_p(au), _p(bu), a.size))
    s = 0.0
    for x, y in zip(a.astype(np.float32), b.astype(np.float32)):
        s = f32emu.add32(s, f32emu.mul32(float(x), float(y)))
    assert got == np.float32(s)


def _planes(r, nplanes, nbytes):
    return r.integers(0, 256, (nplanes, nbytes), dtype=np.uint8)


def _digits(planes):
    bits = np.unpackbits(planes, axis=1, bitorder="little").astype(np.int64)
    return sum(bits[p] << p for p in range(planes.shape[0]))


# x86_64.rs:544-572 / 574-602 / 784-816: sizes 128..1024 bytes per plane (+ edge sizes)
@pytest.mark.parametrize("nbytes", [1, 16, 31, 32, 33, 64, 65, 128, 256, 512, 1024])
def test_subbyte_avx2_equals_scalar_equals_digit_dot(nbytes):
    r = rng(300 + nbytes)
    L = lib()
    for res, sc, av in ((1, L.orc_dot_binary_scalar, L.orc_dot_binary_avx2),
                        (2, L.orc_dot_quaternary_scalar, L.orc_dot_quaternary_avx2),
                        (3, L.orc_dot_octal_scalar, L.orc_dot_octal_avx2)):
        x, y = _planes(r, res, nbytes), _planes(r, res, nbytes)
        s, v = sc(_p(x), _p(y), nbytes), av(_p(x), _p(y), nbytes)
        want = int((_digits(x) * _digits(y)).sum())
        assert s == v == float(want)


def test_quaternary_vs_theoretical_like_reference_test():
    # x86_64.rs:454-505 with a fixed seed: digits 0..3, length 32
    r = rng(42)
    for _ in range(50):
        a = r.integers(0, 4, 32)
        b = r.integers(0, 4, 32)
        va = np.zeros((2, 8), dtype=np.uint8)
        vb = np.zeros((2, 8), dtype=np.uint8)
        for i, (x, y) in enumerate(zip(a, b)):
            bi, off = i // 4, (i % 4) * 2
            va[0, bi] |= (x & 1) << off
            va[1, bi] |= ((x >> 1) & 1) << off
            vb[0, bi] |= (y & 1) << off
            vb[1, bi] |= ((y >> 1) & 1) << off
        got = lib().orc_dot_quaternary_scalar(_p(va), _p(vb), 8)
        assert got == float((a * b).sum())


def test_count_ones_256():
    # x86_64.rs:673-746: simple / random / edge / incremental
    L = lib()
    r = rng(9)
    cases = [np.zeros(32, np.uint8), np.full(32, 0xFF, np.uint8), np.full(32, 0xAA, np.uint8)]
    cases += [r.integers(0, 256, 32, dtype=np.uint8) for _ in range(100)]
    for i in range(33):
        c = np.zeros(32, np.uint8)
        c[:i] = 0xFF
        cases.append(c)
    for c in cases:
        assert L.orc_count_ones_256(_p(c)) == int(np.unpackbits(c).sum())


# ----------------------------------------------------------------- quantization

def test_quantize_u8_formula_and_mag():
    r = rng(11)
    v = np.concatenate([r.uniform(-1.5, 1.5, 500), [-1.0, 1.0, 0.0, -2.0, 2.0, np.nan]]).astype(np.float32)
    lo, hi = np.float32(-1.0), np.float32(1.0)
    code, mag = orc.quantize(orc.ST_U8, v, lo, hi)
    c = np.where(np.isnan(v), lo, np.minimum(np.maximum(v, lo), hi)).astype(np.float32)
    t = ((c - lo) / np.float32(hi - lo)) * np.float32(255.0)
    want = np.trunc(t).astype(np.int64).clip(0, 255).astype(np.uint8)
    assert np.array_equal(code, want)
    ss = int((want.astype(np.uint64) ** 2).sum()) & 0xFFFFFFFF
    assert mag == np.sqrt(np.float32(ss))


@pytest.mark.parametrize("res", [1, 2, 3])
def test_quantize_subbyte_plane_order_and_edge_values(res):
    r = rng(12 + res)
    v = np.concatenate([r.uniform(-1, 1, 61), [-1.0, 1.0, 0.999999, -1.5, 1.5, 0.0, -0.0]]).astype(np.float32)
    code, mag = orc.quantize(res, v)
    nb = (v.size + 7) // 8
    planes = code.reshape(res, nb)
    step = np.float32(2.0) / np.float32(2 ** res)
    t = np.floor((v + np.float32(1.0)) / step)
    n = np.where(t <= 0, 0, t).astype(np.uint64)          # saturating `as usize`
    bits = np.unpackbits(planes, axis=1, bitorder="little")[:, : v.size]
    for p in range(res):                                   # plane 0 = MSB of the low `res` bits
        assert np.array_equal(bits[p], ((n >> np.uint64(res - 1 - p)) & np.uint64(1)).astype(np.uint8))
    # 1.0 wraps to 0, -1.5 saturates to 0 (common.rs:225-236)
    i1 = 62
    assert all(bits[p][i1] == 0 for p in range(res))
    assert mag == orc.mag_f32(v)


def test_quantize_f16_f32():
    v = rng(14).uniform(-1, 1, 100).astype(np.float32)
    code, mag = orc.quantize(orc.ST_F16, v)
    assert np.array_equal(code.view(np.uint16), v.astype(np.float16).view(np.uint16))
    assert mag == orc.mag_f32(v)
    code, mag = orc.quantize(orc.ST_F32, v)
    assert np.array_equal(code.view(np.float32), v)


# -------------------------------------------------------------------- distances

def _q(st, v):
    return orc.quantize(st, v)


@pytest.mark.parametrize("st", range(6))
def test_cosine_formula_and_zero_norm_error(st):
    r = rng(20 + st)
    dim = 100
    x, y = r.uniform(-1, 1, dim).astype(np.float32), r.uniform(-1, 1, dim).astype(np.float32)
    (xc, xm), (yc, ym) = _q(st, x), _q(st, y)
    rc, cs = orc.distance(orc.METRIC_COSINE, st, dim, xc, xm, yc, ym)
    assert rc == orc.OK
    rc2, dp = (orc.OK, orc.dot_f32_simd(x, y)) if st == orc.ST_F32 else orc.distance(orc.METRIC_DOT, st, dim, xc, xm, yc, ym)
    assert rc2 == orc.OK
    assert cs == np.float32(dp) / (np.float32(xm) * np.float32(ym))
    rc, _ = orc.distance(orc.METRIC_COSINE, st, dim, xc, 0.0, yc, ym)
    assert rc == orc.CALCULATION_ERROR           # cosine.rs:230-231


def test_metric_storage_arms_match_reference_table():
    dim = 16
    v = rng(30).uniform(-1, 1, dim).astype(np.float32)
    for st in range(6):
        c, m = _q(st, v)
        rc_dot, _ = orc.distance(orc.METRIC_DOT, st, dim, c, m, c, m)
        rc_eu, _ = orc.distance(orc.METRIC_EUCLIDEAN, st, dim, c, m, c, m)
        rc_ham, _ = orc.distance(orc.METRIC_HAMMING, st, dim, c, m, c, m)
        assert rc_dot == (orc.STORAGE_MISMATCH if st == orc.ST_F32 else orc.OK)      # dotproduct.rs:62
        assert rc_eu == {0: orc.OK, 4: orc.OK, 5: orc.STORAGE_MISMATCH}.get(st, orc.UNIMPLEMENTED)  # euclidean.rs:17-39
        assert rc_ham == (orc.STORAGE_MISMATCH if st == orc.ST_F32 else orc.OK)      # hamming.rs:21-57


def test_euclidean_u8_i16_wrap_and_f16():
    x = np.array([255, 0, 10, 200], dtype=np.uint8)
    y = np.array([0, 255, 10, 19], dtype=np.uint8)
    rc, d = orc.distance(orc.METRIC_EUCLIDEAN, orc.ST_U8, 4, x, 1.0, y, 1.0)
    # 255^2 = 65025 wraps to -511 as i16 (release build), 181^2 = 32761 fits
    want = np.float32(-511.0) + np.float32(-511.0) + np.float32(0.0) + np.float32(32761.0)
    assert rc == orc.OK and d == np.sqrt(np.float32(want))
    x = np.array([255, 0], dtype=np.uint8)
    y = np.array([0, 255], dtype=np.uint8)
    rc, d = orc.distance(orc.METRIC_EUCLIDEAN, orc.ST_U8, 2, x, 1.0, y, 1.0)
    assert rc == orc.OK and np.isnan(d)                                         # sqrt(-1022)
    r = rng(31)
    a, b = r.uniform(-1, 1, 50).astype(np.float16), r.uniform(-1, 1, 50).astype(np.float16)
    rc, d = orc.distance(orc.METRIC_EUCLIDEAN, orc.ST_F16, 50, a.view(np.uint16), 1.0, b.view(np.uint16), 1.0)
    s = 0.0
    for p, q in zip(a.astype(np.float32), b.astype(np.float32)):
        df = f32emu.add32(float(p), -float(q))
        s = f32emu.add32(s, f32emu.mul32(df, df))
    assert d == np.sqrt(np.float32(s))


def test_hamming_subbyte_res3_ignores_top_two_bits():
    x = np.zeros((3, 4), dtype=np.uint8)
    y = np.full((3, 4), 0xFF, dtype=np.uint8)
    rc, d = orc.distance(orc.METRIC_HAMMING, orc.ST_SUB3, 32, x, 1.0, y, 1.0)
    assert rc == orc.OK and d == 3 * 4 * 6          # hamming.rs:86-93: 8/3 = 2 fields of 3 bits
    rc, d = orc.distance(orc.METRIC_HAMMING, orc.ST_SUB2, 32, x[:2], 1.0, y[:2], 1.0)
    assert d == 2 * 4 * 8
    rc, d = orc.distance(orc.METRIC_HAMMING, orc.ST_U8, 4, x[0], 1.0, y[0], 1.0)
    assert d == 32


# --------------------------------------------------------------------- ordering

def test_metric_result_ordering_like_reference_test():
    vals = [6.0, 5.0, 4.0, 3.0, 2.0, 1.0]
    assert sorted(vals, key=lambda v: orc.order_key(orc.METRIC_COSINE, v)) == [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]
    # distance-like metrics are reversed (types.rs:405-407)
    assert sorted(vals, key=lambda v: orc.order_key(orc.METRIC_EUCLIDEAN, v)) == vals
    # total_cmp: -nan < -inf < -1 < -0 < +0 < 1 < inf < +nan
    neg_nan = struct.unpack("<f", struct.pack("<I", 0xFFC00000))[0]
    pos_nan = struct.unpack("<f", struct.pack("<I", 0x7FC00000))[0]
    seq = [neg_nan, -math.inf, -1.0, -0.0, 0.0, 1.0, math.inf, pos_nan]
    keys = [orc.order_key(orc.METRIC_COSINE, v) for v in seq]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)


# ------------------------------------------------------------- brute / re-rank

def test_brute_topk_f32_matches_numpy_ground_truth_procedure():
    # tests/test-dataset.py:312-316: normalise rows, matrix product, top-k
    corpus = orc.synth_matrix(3, 2000, 64)
    queries = orc.synth_matrix(4, 8, 64)
    ids, scores = orc.brute_topk_f32(corpus, queries, 10, threads=4)
    a = corpus / np.linalg.norm(corpus, axis=1, keepdims=True)
    b = queries / np.linalg.norm(queries, axis=1, keepdims=True)
    sim = (b.astype(np.float64) @ a.astype(np.float64).T)
    want = np.argsort(-sim, axis=1)[:, :10]
    assert np.array_equal(ids, want.astype(np.uint32))
    assert np.allclose(scores, np.take_along_axis(sim, want, axis=1), rtol=1e-5, atol=1e-6)
    # score == per-pair finalize formula
    for qi in range(8):
        mq = orc.mag_f32(queries[qi])
        for j in range(10):
            v = corpus[ids[qi, j]]
            assert scores[qi, j] == orc.dot_f32_simd(queries[qi], v) / (mq * orc.mag_f32(v))


def test_brute_topk_tie_rule_and_short_corpus():
    corpus = np.tile(orc.synth_matrix(5, 1, 16), (6, 1))
    q = orc.synth_matrix(6, 1, 16)
    ids, scores = orc.brute_topk_f32(corpus, q, 4)
    assert ids.tolist() == [[0, 1, 2, 3]]               # equal scores -> smaller id first
    ids, scores = orc.brute_topk_f32(corpus[:2], q, 4)
    assert ids.tolist() == [[0, 1, 0xFFFFFFFF, 0xFFFFFFFF]]


def test_rerank_matches_brute_on_candidates():
    corpus = orc.synth_matrix(7, 500, 48)
    q = orc.synth_matrix(8, 1, 48)[0]
    cand = np.array([5, 499, 17, 250, 3, 77, 78], dtype=np.uint32)
    ids, scores = orc.rerank_f32(corpus, q, cand, 3)
    full_ids, full_scores = orc.brute_topk_f32(corpus[cand], q[None], 3)
    assert np.array_equal(ids, cand[full_ids[0]])
    assert np.array_equal(scores, full_scores[0])


def test_brute_codes_zero_norm_sets_error_flag():
    dim = 32
    m = orc.synth_matrix(9, 20, dim)
    m[7] = 0.0
    codes, mags = orc.quantize_batch(orc.ST_SUB2, m)
    qc, qm = orc.quantize_batch(orc.ST_SUB2, orc.synth_matrix(10, 2, dim))
    rc, ids, scores, err = orc.brute_topk_codes(orc.METRIC_COSINE, orc.ST_SUB2, dim, codes, mags, qc, qm, 5)
    assert rc == 0 and err.tolist() == [1, 1] and 7 not in ids
    rc, ids, scores, err = orc.brute_topk_codes(orc.METRIC_DOT, orc.ST_SUB2, dim, codes, mags, qc, qm, 5)
    assert rc == 0 and err.tolist() == [0, 0]


# ------------------------------------------------------------------ bfloat16 (labelled extension, ST_BF16)
def test_bf16_extension_conversion_and_dot_against_independent_restatements():
    """not a reference storage type: what HalfPrecisionFP would compute with half::bf16.  Conversion = round to nearest
    even on the upper 16 bits (NaN keeps its sign, quiet bit set); dot = sequential f32 fold of exact products."""
    rng = np.random.default_rng(77)
    v = np.concatenate([rng.normal(size=4000).astype(np.float32), orc.synth_matrix(5, 1, 4000)[0],
                        np.array([0.0, -0.0, 1.0, -1.0, 1e-40, -1e-40, 3.3895314e38, np.inf, -np.inf, 65504.0,
                                  1.00390625, 1.005859375, 1.01171875], dtype=np.float32)])
    code, mag = orc.quantize_batch(orc.ST_BF16, v[None])
    got = code.view(np.uint16)[0]
    x = v.view(np.uint32).astype(np.uint64)
    want = ((x + 0x7FFF + ((x >> 16) & 1)) >> 16).astype(np.uint16)          # RNE restated arithmetically
    assert np.array_equal(got, want)
    bits = lambda a_: np.ascontiguousarray(a_, dtype=np.float32).view(np.uint32)
    nan = np.array([np.float32("nan"), -np.float32("nan")], dtype=np.float32)
    ncode, _ = orc.quantize_batch(orc.ST_BF16, nan[None])
    nb = ncode.view(np.uint16)[0]
    assert ((nb & 0x7F80) == 0x7F80).all() and ((nb & 0x0040) != 0).all() and (nb[0] >> 15) != (nb[1] >> 15)
    # dot: exact products (8-bit significands), sequential f32 adds
    a, b = orc.synth_matrix(6, 1, 333)[0], orc.synth_matrix(7, 1, 333)[0]
    ac, am = orc.quantize_batch(orc.ST_BF16, a[None])
    bc, bm = orc.quantize_batch(orc.ST_BF16, b[None])
    fa = (ac.view(np.uint16)[0].astype(np.uint32) << 16).view(np.float32)
    fb = (bc.view(np.uint16)[0].astype(np.uint32) << 16).view(np.float32)
    s = np.float32(0)
    for i in range(333):
        p = np.float64(fa[i]) * np.float64(fb[i])
        assert np.float64(np.float32(p)) == p                                # the product is exact in f32
        s = np.float32(s + np.float32(p))
    rc, d = orc.distance(orc.METRIC_DOT, orc.ST_BF16, 333, ac[0], am[0], bc[0], bm[0])
    assert rc == orc.OK and bits(np.array([d], np.float32))[0] == bits(np.array([s], np.float32))[0]
    rc, c = orc.distance(orc.METRIC_COSINE, orc.ST_BF16, 333, ac[0], am[0], bc[0], bm[0])
    assert rc == orc.OK and bits(np.array([c], np.float32))[0] == bits(np.array([s / np.float32(am[0] * bm[0])], np.float32))[0]


def test_fused_multiply_add_of_16_bit_operands_equals_the_reference_fold():
    """The CUDA kernels fold f16 / bf16 dot products with ONE fused multiply-add per element (operands widened exactly to
    f32, a*b + c rounded once).  The reference rounds twice (f32 multiply, then f32 add).  Both
    agree because the product of two halfs (11-bit significands) or two bf16 values (8-bit) is exact in f32 -- checked here
    with the exact-integer binary32 emulation over operands that include subnormals, the largest finite values and sign
    mixes, against the oracle's dot_product_f16 / bf16 arm."""
    r = rng(66)
    L = lib()
    # halfs: random normals, subnormals (|x| < 2^-14), the extremes
    raw = np.concatenate([r.uniform(-1, 1, 400), r.uniform(-6e-5, 6e-5, 120), r.uniform(-6e-8, 6e-8, 40),
                          [65504.0, -65504.0, 6.1e-5, -6.1e-5, 5.96e-8, 0.0, -0.0, 1.0, -1.0, 0.333251953125]])
    a = raw.astype(np.float16)
    b = r.permutation(raw).astype(np.float16)
    assert (np.abs(a.astype(np.float32)) < 6.1e-5).sum() > 100              # subnormal halfs present
    fused = two = 0.0
    for x, y in zip(a.astype(np.float32), b.astype(np.float32)):
        p = f32emu.mul32(float(x), float(y))
        assert p == float(np.float64(x) * np.float64(y))                    # exact product, also for subnormal operands
        fused = f32emu.fma32(float(x), float(y), fused)
        two = f32emu.add32(two, p)
        assert fused == two
    got = np.float32(L.orc_dot_f16(_p(a.view(np.uint16)), _p(b.view(np.uint16)), a.size))
    assert got == np.float32(fused)
    # bf16: same statement with 8-bit significands and the f32 exponent range (products can overflow / underflow like any f32 product)
    v = np.concatenate([r.normal(size=300).astype(np.float32), np.array([3.0e38, -3.0e38, 1e-38, -1e-38, 1e-40, 1.0, -0.0], np.float32)])
    ca, ma = orc.quantize_batch(orc.ST_BF16, v[None])
    cb, mb = orc.quantize_batch(orc.ST_BF16, r.permutation(v)[None])
    fa = (ca.view(np.uint16)[0].astype(np.uint32) << 16).view(np.float32)
    fb = (cb.view(np.uint16)[0].astype(np.uint32) << 16).view(np.float32)
    fused = two = 0.0
    finite = True
    for x, y in zip(fa, fb):
        if not (np.isfinite(fused) and np.isfinite(two)):
            finite = False
            break
        p64 = np.float64(x) * np.float64(y)
        if abs(p64) >= 2.0 ** 128 or (p64 != 0 and abs(p64) < 2.0 ** -126):
            continue                                                        # products outside the normal f32 range round in both forms; skipped
        fused = f32emu.fma32(float(x), float(y), fused)
        two = f32emu.add32(two, f32emu.mul32(float(x), float(y)))
        assert fused == two
    assert finite
