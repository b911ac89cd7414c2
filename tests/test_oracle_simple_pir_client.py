"""The seeded client reference (tests/simple_pir_client_ref.py) against the oracle: its noiselessSample through the
materialised A equals the reference's polynomial form, and its wrapped results equal the exact product wherever the
double-width sum stays below 2^(2 word_bits)."""
import numpy as np
import pytest

import simple_pir_client_ref as ref
from oracle import simple_pir_oracle as osp


@pytest.mark.parametrize("n,k,cpe", [(8, 7, 1), (16, 37, 3), (16, 50, 2)])
def test_seeded_noiseless_sample_matches_the_polynomial_form(n, k, cpe):
    p = osp.ntt_friendly_mod(28, n)
    s = ref.secrets_from_seed(bytes([n, k, cpe]) * 8 + bytes(8), cpe, n)
    assert set(np.unique(s)) <= {-1, 0, 1}
    polys = osp.a_polynomials(bytes(32), n, -(-k // n), p)
    assert np.array_equal(osp.noiseless_sample(s, osp.a_matrix(polys, k, p), p),
                          osp.noiseless_sample_polynomial(s, polys, k, p))


@pytest.mark.parametrize("w,ct,n", [(32, 20, 16), (32, 28, 64), (64, 42, 2048)])
def test_wrapped_results_equal_exact_where_the_sum_does_not_wrap(w, ct, n):
    p = osp.ntt_friendly_mod(ct, n)
    rng = np.random.default_rng(ct)
    hint = rng.integers(0, p, size=(9, n), dtype=np.uint64)
    s = ref.secrets_from_seed(bytes(range(32)), 2, n)
    pos, neg = ref.exact_products(s, hint)
    no_wrap = (pos + (p - 1) * neg) < (1 << (2 * w))
    wrapped, exact = ref.results(s, hint, p, w), ref.results(s, hint, p, w, exact=True)
    assert np.array_equal(wrapped[no_wrap], exact[no_wrap])
    if w == 64:
        assert no_wrap.all()
