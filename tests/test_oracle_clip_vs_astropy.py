"""Pins tests/_cdpp_oracle.sigma_clip_mask with asymmetric sigma_lower / sigma_upper, and maxiters=None, against REAL
astropy when it is importable (skipped otherwise, like tests/test_oracle_vs_astropy.py)."""
import os
import sys

import numpy as np
import pytest

astropy = pytest.importorskip("astropy", reason="astropy is not installed here")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _cdpp_oracle as O  # noqa: E402


@pytest.mark.parametrize("sigma_lower,sigma_upper,maxiters", [(2.0, 4.0, 5), (4.0, 2.0, 5), (np.inf, 3.0, 5),
                                                              (3.0, np.inf, None), (3.0, 3.0, None)])
def test_asymmetric_sigma_clip_mask_matches_astropy(sigma_lower, sigma_upper, maxiters):
    from astropy.stats import sigma_clip
    rng = np.random.default_rng(12)
    x = rng.normal(size=20000)
    x[rng.choice(20000, 200, replace=False)] += rng.exponential(6.0, 200)
    for s in rng.choice(19960, 40, replace=False):
        x[s:s + 30] -= np.exp(rng.uniform(np.log(2.0), np.log(80.0)))
    x[::997] = np.nan
    x[5::1999] = np.inf
    ref = np.ma.getmaskarray(sigma_clip(x, sigma_lower=sigma_lower, sigma_upper=sigma_upper, maxiters=maxiters))
    got = O.sigma_clip_mask(x, sigma_lower=sigma_lower, sigma_upper=sigma_upper, maxiters=maxiters)
    np.testing.assert_array_equal(got, ref)
