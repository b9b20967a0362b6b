"""Executable statement of the residual term of the MaxSim filter's certificate (k_maxsim_tc, DESIGN.md 4c).
The tensor cores take q.w from fp16 operands: the query row scaled by 2^qexp (qexp = -ilogb(|q|max), so the largest
scaled row norm is in [1, 2)), the bucket weights as they are; products are exact, sums are fp32; the result is scaled
back by 2^-qexp.  The certificate charges this term

    |q.w - 2^-qexp h(2^qexp q).h(w)| <= |q|max wmax (2u + u^2 + 2^-15)        (u = 2^-11)

where 2u + u^2 is the relative rounding of the two operands, and 2^-15 the fp16 subnormal spacing (absolute 2^-25 per
coordinate against a scaled norm >= 1) plus the fp32 accumulation (dim 2^-24).  Pure numpy: fp16 operands, float64
accumulation, plus the worst case of the fp32 accumulator.  Without the scaling the same statement fails for small
queries (coordinates in the fp16 subnormal range) and for a coordinate of 1e5 (fp16 overflow): the model is not vacuous."""
import numpy as np
import pytest

U = 2.0 ** -11


def _setup(dim, nbits, seed=0, n_tok=300, nq=16):
    rng = np.random.default_rng(seed + 7 * dim + nbits)
    w = (0.05 * np.linspace(-1.8, 1.8, 1 << nbits)).astype(np.float32)
    W = w[rng.integers(0, 1 << nbits, (n_tok, dim))]                       # the residual vectors of the tokens
    Q = rng.standard_normal((nq, dim)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return W, Q.astype(np.float32)


def _worst_ratio(Q, W, scaled):
    """Largest residual-term error over every (query token, token) pair / its share of eps_q."""
    Q64, W64 = Q.astype(np.float64), W.astype(np.float64)
    qmax = np.linalg.norm(Q64, axis=1).max()
    wmax = np.linalg.norm(W64, axis=1).max()
    kq = -int(np.floor(np.log2(qmax))) if scaled else 0          # -ilogb(|q|max), as k_query_range computes it
    with np.errstate(over="ignore"):
        hq = np.ldexp(Q, kq).astype(np.float32).astype(np.float16).astype(np.float64)   # exact scaling, then fp16
    hw = W.astype(np.float16).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        acc = hq @ hw.T                                           # exact products, float64 sums
        fp32_term = W.shape[1] * 2.0 ** -24 * (np.abs(hq) @ np.abs(hw).T)   # fp32 accumulation, worst case
        err = np.abs(np.ldexp(acc, -kq) - Q64 @ W64.T) + np.ldexp(fp32_term, -kq)
    share = qmax * wmax * (2 * U + U * U + 2.0 ** -15)
    err = np.where(np.isfinite(err), err, np.inf)
    return float(err.max() / share)


SCALES = [1e-30, 1e-20, 1e-12, 1e-8, 1e-6, 1e-5, 1e-4, 1e-2, 1.0, 4096.0, 1e5, 1e8, 1e20, 1e30]


@pytest.mark.parametrize("dim", [64, 96, 128])
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_scaled_operand_keeps_the_residual_term_within_its_share(dim, nbits):
    W, Q = _setup(dim, nbits)
    ratios = []
    for s in SCALES:
        r = _worst_ratio((Q * np.float32(s)).astype(np.float32), W, scaled=True)
        assert r <= 1.0, (dim, nbits, s, r)
        ratios.append(r)
    assert max(ratios) > 0.01                         # the bound is not loose by orders of magnitude
    big = Q.copy()
    big[0, 3] = 1e5                                   # one coordinate of 1e5 in an otherwise unit query
    assert _worst_ratio(big, W, scaled=True) <= 1.0


@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("nbits", [2, 4])
def test_raw_operand_breaks_the_bound_for_small_and_large_queries(dim, nbits):
    W, Q = _setup(dim, nbits)
    assert _worst_ratio(Q, W, scaled=False) <= 1.0                       # unit queries are fine either way
    assert _worst_ratio((Q * np.float32(1e-6)).astype(np.float32), W, scaled=False) > 1.0   # fp16 subnormals
    big = Q.copy()
    big[0, 3] = 1e5
    assert _worst_ratio(big, W, scaled=False) == np.inf                  # fp16 overflow: a non-finite estimate
