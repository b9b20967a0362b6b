"""The MaxSim filter's certificate measured on the device (k_maxsim_tc; DESIGN.md 4c).  Every similarity estimate of
the filter must lie within eps_q = |q|max * eps_unit of the exact one, or a doc (pass 1) or a (token, query token) pair
(pass 2) that holds a result is dropped.  PB_FILTER_DIAG=1 scores every kept doc exactly and reports the largest
|pass-1 estimate maximum - exact maximum| / eps_q (filter_err_ratio_e6, in millionths): here it must stay <= 1 on the
tensor-core table, the exact table and without a table, over dims, bit widths, query shapes and scales, and indexes
with extreme constants.  Then near ties built in the codec domain -- docs and tokens whose exact scores sit inside the bands -- must come out bit for bit as
the CPU oracle's while the filter really decides them."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODES = {"linear_tc_table": {}, "linear_exact_table": {"PB_K1_TC": "0"}, "no_score_table": {"PB_FAST_APPROX": "0"}}
KW = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None)   # any query scale finds candidates
ENVS = ("PB_FILTER_DIAG", "PB_K1_TC", "PB_FAST_APPROX")


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _open(npb, ix, monkeypatch, env):
    """Open with `env` set (the handle reads it at open) and nothing else of ENVS."""
    for k in ENVS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths,
                                         ix.ivf, ix.ivf_lengths, ix.nbits)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def _same(a, w):
    return a.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(a.scores, w.scores, equal_nan=True)


def _codec_index(oracle, dim=128, nbits=4, K=256, D=400, T=24, seed=5, wscale=0.05, cscale=1.0):
    """Random unit centroids (times cscale), random residual bytes, bucket weights wscale * linspace(-1.8, 1.8)."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cent = (cent * np.float32(cscale)).astype(np.float32)
    codes = rng.integers(0, K, D * T).astype(np.int64)
    res = rng.integers(0, 256, (D * T, dim * nbits // 8), dtype=np.uint8)
    w = (wscale * np.linspace(-1.8, 1.8, 1 << nbits)).astype(np.float32)
    dl = rng.integers(T // 2, T + 1, D).astype(np.int64)
    codes, res = codes[:dl.sum()], res[:dl.sum()]
    ivf, lens = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, None, codes, res, dl, ivf, lens, nbits)


def _grid(nbits, K, dim, rng):
    """Bucket weights on a symmetric grid without 0 (step 0.3 / (2^nbits - 1)), centroids with coordinates on the same
    grid and equal in pairs (2i, 2i + 1): the bucket of -c_i cancels a coordinate exactly, and swapping the residual
    fields of a pair leaves |c + w| unchanged."""
    nb = 1 << nbits
    w = (0.3 / (nb - 1) * (np.arange(nb) - (nb - 1) / 2)).astype(np.float32)
    cut = ((w[1:] + w[:-1]) / 2).astype(np.float32)
    cb = rng.integers(0, nb, (K, dim))
    cb[:, 1::2] = cb[:, 0::2]
    return w, cut, w[cb].astype(np.float32), cb


def _near_cancel(rng, cb, code, nb, n_off=4):
    """Buckets that cancel centroid `code` except at n_off even coordinates, one grid step off: |c + w| = step sqrt(n_off)."""
    b = (nb - 1 - cb[code]).copy()
    for j in 2 * rng.choice(cb.shape[1] // 2, n_off, replace=False):
        b[j] = b[j] + 1 if b[j] < nb - 1 else b[j] - 1
    return b


def _grid_index(oracle, w, cut, cent, docs, nbits):
    """docs = list of [(code, buckets[dim]), ...] -> oracle.Index."""
    codes = np.array([c for d in docs for c, _ in d], np.int64)
    bks = np.stack([b for d in docs for _, b in d])
    res = oracle.quantize_residuals(w[bks].astype(np.float32), cut, nbits)
    dl = np.array([len(d) for d in docs], np.int64)
    ivf, lens = oracle.build_ivf(codes, dl, cent.shape[0])
    return oracle.Index(cent, w, cut, codes, res, dl, ivf, lens, nbits)


def _queries(rng, dim, nq, n):
    q = rng.standard_normal((n, nq, dim)).astype(np.float32)
    return [(x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32) for x in q]


def _scaled_batch(qs):
    """Every query of qs at every scale of the diagnostic, and one with a coordinate of 1e5."""
    out = []
    for i, q in enumerate(qs):
        for s in (1e-8, 1e-6, 1e-4, 1.0, 4096.0, 1e6):
            out.append((q * np.float32(s)).astype(np.float32))
        big = q.copy()
        big[0, i % q.shape[1]] = 1e5
        out.append(big)
    return out


def _check_diag(npb, gpu, batch, what):
    gpu.search_batch(batch, npb.SearchParameters(**KW))
    w = gpu.last_work_counters()
    assert w["n_filter_docs"] > 0, (what, w)                  # the filter ran: a case that turns it off fails
    assert w["filter_diag_pairs"] > 0, (what, w)
    assert 0 < w["filter_err_ratio_e6"] <= 1_000_000, (what, w["filter_err_ratio_e6"])
    return w


def _diag_all_modes(npb, oracle, ix, monkeypatch, what, check_results=False):
    rng = np.random.default_rng(len(what))
    base = [q for n in (1, 32, 33, 64) for q in _queries(rng, ix.dim, n, 1)]
    for mode, env in MODES.items():
        gpu = _open(npb, ix, monkeypatch, dict(env, PB_FILTER_DIAG="1"))
        try:
            for lo, hi in ((0, 2), (2, 4)):   # nq <= 32 (N = 32 operand) and 33 / 64 (N = 64)
                batch = _scaled_batch(base[lo:hi])
                _check_diag(npb, gpu, batch, (what, mode, lo))
                if check_results and mode == "linear_tc_table":
                    res = gpu.search_batch(batch[:7], npb.SearchParameters(**KW))
                    po = oracle.SearchParameters(**KW)
                    for q, r in zip(batch[:7], res):
                        assert _same(r, oracle.search_one(ix, q, po)), (what, mode)
        finally:
            gpu.close()


@pytest.mark.parametrize("dim", [64, 96, 128])
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_filter_estimate_is_within_its_certificate_on_codec_indexes(npb, oracle, monkeypatch, dim, nbits):
    ix = _codec_index(oracle, dim=dim, nbits=nbits, seed=dim + nbits)
    _diag_all_modes(npb, oracle, ix, monkeypatch, f"codec d{dim} b{nbits}")


@pytest.fixture(scope="module")
def oracle_index(oracle):
    docs = oracle.synthetic_corpus(400, 30, dim=128, seed=17, ragged=True)
    return oracle.create_index(docs, nbits=4, seed=3, num_partitions=256)


def test_filter_estimate_is_within_its_certificate_on_an_oracle_index(npb, oracle, monkeypatch, oracle_index):
    _diag_all_modes(npb, oracle, oracle_index, monkeypatch, "oracle", check_results=True)


@pytest.mark.parametrize("kind", ["near_cancelling", "subnormal_weights", "centroid_norm_1e3"])
def test_filter_estimate_is_within_its_certificate_at_extreme_index_constants(npb, oracle, monkeypatch, kind):
    if kind == "near_cancelling":
        # a quarter of the tokens nearly cancel their centroid: min |c + w| = 0.04, eps_unit just under 0.05
        rng = np.random.default_rng(7)
        nbits, K, dim = 4, 64, 128
        w, cut, cent, cb = _grid(nbits, K, dim, rng)
        docs = []
        for _ in range(400):
            d = []
            for _ in range(int(rng.integers(8, 25))):
                c = int(rng.integers(K))
                b = _near_cancel(rng, cb, c, 1 << nbits) if rng.random() < 0.25 else rng.integers(0, 1 << nbits, dim)
                d.append((c, b))
            docs.append(d)
        ix = _grid_index(oracle, w, cut, cent, docs, nbits)
    elif kind == "subnormal_weights":
        ix = _codec_index(oracle, wscale=1e-5, seed=31)      # every bucket weight is an fp16 subnormal
    else:
        ix = _codec_index(oracle, cscale=1e3, wscale=50.0, seed=32)
    _diag_all_modes(npb, oracle, ix, monkeypatch, kind)


def test_filter_estimate_is_within_its_certificate_after_append_and_delete(npb, oracle, monkeypatch, oracle_index):
    ix = oracle_index
    w = ix.bucket_weights
    rng = np.random.default_rng(12)
    far = int(np.argmax(np.abs(w)))
    n_codes = rng.integers(0, ix.num_centroids, 40)
    rows = oracle.quantize_residuals(np.full((40, ix.dim), w[far], np.float32), ix.bucket_cutoffs, ix.nbits)
    dl_new = np.array([1, 4, 35], np.int64)
    rng2 = np.random.default_rng(4)
    base = [q for n in (1, 32, 33, 64) for q in _queries(rng2, ix.dim, n, 1)]
    for mode, env in MODES.items():
        gpu = _open(npb, ix, monkeypatch, dict(env, PB_FILTER_DIAG="1"))
        try:
            gpu.append_encoded(n_codes, rows, dl_new)          # every field in the largest-|weight| bucket: wmax rises
            for lo, hi in ((0, 2), (2, 4)):
                _check_diag(npb, gpu, _scaled_batch(base[lo:hi]), ("append", mode, lo))
            gpu.delete(list(range(0, ix.num_documents, 3)) + [ix.num_documents + 2])
            for lo, hi in ((0, 2), (2, 4)):
                _check_diag(npb, gpu, _scaled_batch(base[lo:hi]), ("delete", mode, lo))
        finally:
            gpu.close()


# ------------------------------------------------------------------------------------------
# near ties the filter has to decide
# ------------------------------------------------------------------------------------------
def _straddle(q):
    """Put the coordinates of every pair (2i, 2i + 1) one fp32 ulp either side of the same fp16 rounding midpoint:
    q_2i > q_2i+1 by two fp32 ulps, but fp16 rounds them a whole fp16 ulp apart, the other way round relative to
    the grid -- the estimate sees a difference the exact dot does not."""
    q = q.astype(np.float32).copy()
    x = q[:, 0::2]
    h = x.astype(np.float16)
    nxt = np.nextafter(h, np.where(x >= 0, np.float16(np.inf), np.float16(-np.inf))).astype(np.float32)
    m = ((h.astype(np.float32) + nxt) / 2).astype(np.float32)
    away = np.where(x >= 0, np.float32(np.inf), np.float32(-np.inf))
    q[:, 0::2] = np.nextafter(m, away)
    q[:, 1::2] = np.nextafter(m, -away)
    return q


def _swap(rng, b, keep=-1, p=0.5):
    """Swap the fields of a random half of the pairs whose buckets differ (|c + w| is unchanged: c_2i = c_2i+1), all
    but pair `keep`."""
    b = b.copy()
    for i in range(len(b) // 2):
        if i != keep and b[2 * i] != b[2 * i + 1] and rng.random() < p:
            b[2 * i], b[2 * i + 1] = b[2 * i + 1], b[2 * i]
    return b


def _adversarial_small(q, A, B, scale):
    """q * scale with every coordinate just short of a rounding midpoint of the fp16 subnormal grid (spacing 2^-24),
    on the side where fp16(q) - q pushes the estimate of token A down and of token B up.  The linear estimate takes
    the residual part q.w / |v| through fp16 (k_maxsim_tc), so the error of sim~_A - sim~_B is
    sum_i (fp16(q_i) - q_i) (w_A,i / |v_A| - w_B,i / |v_B|).  One coordinate then sets the exact order: A holds the
    maximum by 5 % of the largest error that difference can take.  A = (D, w, |v|) of a token."""
    s = 2.0 ** -24
    (DA, wA, nA), (DB, wB, nB) = A, B
    y = q.astype(np.float64) * scale
    dw = wA / nA - wB / nB
    g = np.floor(y / s)
    y = np.where(dw > 0, (g + 0.5) * s - s / 64, (g + 0.5) * s + s / 64)   # rounds to g s (down) / (g + 1) s (up)
    d = DA - DB
    i = int(np.argmax(np.abs(d)))
    want = 0.05 * 0.5 * s * np.abs(dw).sum()
    y[i] += (want - float(y @ d)) / d[i]
    assert y @ d > 0
    return y.astype(np.float32)


def _tie_case(oracle, kind, seed=0, top_k=10):
    rng = np.random.default_rng(100 + seed)
    nbits, K, dim, nb = 4, 32, 128, 16
    w, cut, cent, cb = _grid(nbits, K, dim, rng)

    def dirn(c, b):
        v = cent[c].astype(np.float64) + w[b]
        return v / np.linalg.norm(v)

    def tok(c, b):
        v = cent[c].astype(np.float64) + w[b]
        return v / np.linalg.norm(v), w[b].astype(np.float64), np.linalg.norm(v)

    nq = 8
    n_cluster = 3 * top_k
    small = kind == "small_norm_adversarial"
    base = []
    for _ in range(nq):
        c = int(rng.integers(K))
        base.append((c, _near_cancel(rng, cb, c, nb) if small else rng.integers(0, nb, dim)))
    # the pair holding the query's 1e5 coordinate is never swapped: the cluster stays inside the band
    keep = [int(np.argmax(dirn(c, b))) // 2 if kind == "coordinate_1e5" else -1 for c, b in base]
    docs = []
    if kind == "one_token_docs":
        for _ in range(n_cluster):
            docs.append([(base[0][0], _swap(rng, base[0][1]))])
        for _ in range(300):
            docs.append([(int(rng.integers(K)), rng.integers(0, nb, dim))])
    else:
        rivals = []
        if small:   # a second near-cancelling token per query token, on another centroid
            for c, _ in base:
                c2 = int((c + 1 + rng.integers(K - 1)) % K)
                rivals.append((c2, _near_cancel(rng, cb, c2, nb)))
        for _ in range(n_cluster):
            d = []
            for t, (c, b) in enumerate(base):
                if small:   # A and its rival compete for query token t; the docs differ in one ordinary token
                    d += [(c, b), rivals[t]]
                    continue
                d.append((c, _swap(rng, b, keep[t])))
                if kind == "competing_tokens":
                    d.append((c, _swap(rng, b, keep[t])))
            if small:
                d.append((int(rng.integers(K)), rng.integers(0, nb, dim)))
            perm_d = rng.permutation(len(d))
            docs.append([d[i] for i in perm_d])
        # at |q| ~ 1e-5 pass 1 keeps every doc and the pair band's absolute 1e-6 lists every token of a filler doc:
        # few fillers, so that the pair list does not overflow and the band itself decides
        for _ in range(40 if small else 300):
            docs.append([(int(rng.integers(K)), rng.integers(0, nb, dim)) for _ in range(nq)])
    perm = rng.permutation(len(docs))
    docs = [docs[i] for i in perm]
    ix = _grid_index(oracle, w, cut, cent, docs, nbits)
    qs = []
    for i in range(6):
        if kind == "one_token_docs":
            D0 = dirn(*base[0])
            q = np.stack([D0 + 0.05 * rng.standard_normal(dim) / np.sqrt(dim) for _ in range(nq)])
        else:
            q = np.stack([dirn(c, b) + 0.05 * rng.standard_normal(dim) / np.sqrt(dim) for c, b in base])
        q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
        if small:
            q = np.stack([_adversarial_small((dirn(*base[t]) + dirn(*rivals[t])) / 2, tok(*base[t]), tok(*rivals[t]),
                                             2.0 ** -(16 + i % 3)) for t in range(nq)])
        else:
            q = _straddle(q)
        if kind == "coordinate_1e5":
            for t in range(nq):
                q[t, int(np.argmax(dirn(*base[t])))] = 1e5
        qs.append(q.astype(np.float32))
    return ix, qs


@pytest.mark.parametrize("kind", ["swapped_fields", "one_token_docs", "competing_tokens", "small_norm_adversarial",
                                  "coordinate_1e5"])
@pytest.mark.parametrize("mode", ["linear_tc_table", "linear_exact_table"])
def test_near_ties_inside_the_bands_match_the_oracle(npb, oracle, monkeypatch, kind, mode):
    top_k = KW["top_k"]
    kw = KW
    if kind == "small_norm_adversarial":   # the probe cannot see near-cancelling tokens: probe and keep every doc
        kw = dict(KW, n_ivf_probe=32, n_full_scores=2048)
    for seed in range(2):
        ix, qs = _tie_case(oracle, kind, seed, top_k)
        gpu = _open(npb, ix, monkeypatch, MODES[mode])
        try:
            res = gpu.search_batch(qs, npb.SearchParameters(**kw))
            w = gpu.last_work_counters()
            po = oracle.SearchParameters(**kw)
            bad = [i for i, (q, r) in enumerate(zip(qs, res)) if not _same(r, oracle.search_one(ix, q, po))]
            assert not bad, (kind, mode, seed, bad)
            w = {k: w[k] for k in ("n_filter_docs", "n_exact_docs", "n_pair_fallback_queries", "n_k1_tc_redo", "n_exact_pairs")}
            w["case"] = (kind, mode, seed)
            assert w["n_filter_docs"] > 0, w
            assert w["n_pair_fallback_queries"] == 0 and w["n_k1_tc_redo"] == 0, w
            assert w["n_exact_docs"] > top_k * len(qs), w          # ties around the top_k-th score were kept
            if kind == "small_norm_adversarial":
                # pass 1 keeps every kept doc at |q| ~ 1e-5: its absolute slack of 1e-3 exceeds any score gap there
                # (DESIGN.md 8); the pair band of pass 2 is what this case tests
                assert w["n_exact_docs"] <= w["n_filter_docs"], w
            else:
                assert w["n_exact_docs"] < w["n_filter_docs"], w
        finally:
            gpu.close()
