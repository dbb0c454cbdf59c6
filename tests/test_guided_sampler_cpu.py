"""CPU: the exact fp32 keys of k_sample's three-row prompt-guidance mix (guidance_scale = (s, p), causal.py:89-105).

k_sample forms, from the fp32 scales s and p it receives through the C ABI, three coefficients in double, each rounded
once to fp32 (as torch does for a Python scalar times an fp32 tensor), then the key in fp32 with this rounding order:
    cb = fp32(s + p - 1), cs = fp32(1 - s), cp = fp32(1 - p)
    k  = fdiv_rn(fadd_rn(fadd_rn(fmul_rn(cb, l_c), fmul_rn(cs, l_u)), fmul_rn(cp, l_p)), max(T, 1e-5))
`keys3` restates this in numpy float32; tests/test_guided_sampler_ops_gpu.py starts its float64 reference from it.
  * Dyadic scales: the coefficients equal those formed from the Python doubles, so keys3 equals torch's own fp32
    evaluation of oracle/prompt_guidance_port.mix3 (then / T) bit for bit.
  * Other scales: s and p are rounded to fp32 before the coefficients are formed.  A coefficient then differs from the
    one formed from the Python doubles by at most ulp(s)/2 + ulp(p)/2 (only the scales it contains) plus half an ulp of
    each rounded coefficient: one fp32 ulp at (3.1, 1.7), more when a scale is close to 1 (1 - s is then much smaller
    than s, 1.1 gives 3 ulps of 1 - s).  The absolute change stays below the rounding of the largest product.
  * The designed-tie inputs the GPU sensitivity checks use are verified here: every key equal under the kernel's
    formula, not under the altered formula.
"""
import numpy as np
import pytest
import torch

from oracle import prompt_guidance_port as G

F32 = np.float32
DYADIC = [(3.0, 2.0), (1.5, 1.5), (1.0, 4.0), (2.5, 3.0), (1.0, 1.0 + 2.0 ** -23)]
NON_DYADIC = [(3.1, 1.7), (1.1, 1.3), (2.7, 1.05)]


def coeffs3(s, p, fp32_sum=False):
    """(cb, cs, cp) as k_sample forms them from the fp32 scales; fp32_sum: the altered formation s + p - 1 in fp32
    (rounded twice) of the sensitivity checks."""
    s32, p32 = F32(s), F32(p)
    if fp32_sum:
        return (s32 + p32) - F32(1), F32(1) - s32, F32(1) - p32
    return F32(float(s32) + float(p32) - 1.0), F32(1.0 - float(s32)), F32(1.0 - float(p32))


def keys3(lc, lu, lp, s, p, T, fp32_sum=False, right_assoc=False):
    """The kernel's fp32 keys [V] from rows cond lc, uncond-speaker lu, uncond-prompt lp.  right_assoc: the altered
    order cb l_c + (cs l_u + cp l_p)."""
    cb, cs, cp = coeffs3(s, p, fp32_sum)
    lc, lu, lp = (np.asarray(x, F32) for x in (lc, lu, lp))
    with np.errstate(invalid="ignore", over="ignore"):
        m = (cb * lc + (cs * lu + cp * lp)) if right_assoc else ((cb * lc + cs * lu) + cp * lp)
        return m / max(F32(T), F32(1e-5))


def _ulps(a, b):
    """Distance in fp32 ulps (both values of one sign)."""
    return abs(int(np.array(a, F32).view(np.int32)) - int(np.array(b, F32).view(np.int32)))


def _ulp(x):
    return float(np.spacing(np.abs(F32(x))))


def tie_rows(s, p, variant):
    """[3, 4096] fp32 rows whose kernel keys (T = 1) are all exactly equal while the altered formula `variant`
    ("fp32_sum" or "right_assoc") splits the even and the odd entries into two key values."""
    cb, cs, cp = coeffs3(s, p)
    rows = np.zeros((3, 4096), F32)
    rows[0, 0::2] = 1.0                                     # even entries: the key is cb itself
    if variant == "fp32_sum":                               # odd entries: cs * w == cb exactly, w within 8 ulps of cb / cs
        w0 = F32(cb / cs)
        near = [w0]
        for d in (F32(np.inf), F32(-np.inf)):
            w = w0
            for _ in range(8):
                w = np.nextafter(w, d)
                near.append(w)
        rows[1, 1::2] = next(w for w in near if cs * w == cb)
    else:                                                   # odd entries: two half-ulp terms that each round back to cb
        e = _ulp(cb) / 2                                    # (ties to even) but round up once summed first
        rows[0, 1::2] = 1.0
        rows[1, 1::2] = e / float(cs)
        rows[2, 1::2] = e / float(cp)
    return rows


@pytest.mark.parametrize("s,p", DYADIC)
@pytest.mark.parametrize("T", [1.0, 0.7, 1e-6])
def test_keys_equal_torch_mix3_for_dyadic_scales(s, p, T):
    rng = np.random.default_rng(int(s * 8 + p * 64))
    V = 4099
    lg = (rng.standard_normal((3, V)) * rng.choice([0.5, 4.0, 40.0], (3, V))).astype(F32)
    lg[:, :64] = rng.choice(np.arange(-8, 9) / 4.0, (3, 64))     # exact products, ties
    assert coeffs3(s, p) == tuple(F32(c) for c in (s + p - 1, 1 - s, 1 - p))
    mixed = G.mix3(torch.from_numpy(lg), s, p)
    assert mixed.dtype == torch.float32
    t = torch.tensor(T, dtype=torch.float32)
    want = (mixed / torch.max(t, 1e-5 * torch.ones_like(t))).numpy()
    got = keys3(lg[0], lg[1], lg[2], s, p, T)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), f"(s, p) = ({s}, {p}), T = {T}"
    if T == 1.0:
        assert np.array_equal(keys3(lg[0], lg[1], lg[2], s, p, 1.0).view(np.int32), mixed.numpy().view(np.int32))


@pytest.mark.parametrize("s,p", NON_DYADIC)
def test_coefficients_for_non_dyadic_scales(s, p):
    """Against the coefficients formed from the Python doubles (torch's): the bound of the module docstring, and one
    ulp exactly where the kernel's comment promises it (3.1, 1.7); the keys follow within one rounding per term."""
    got = coeffs3(s, p)
    py = (F32(s + p - 1), F32(1 - s), F32(1 - p))
    ds, dp = abs(float(F32(s)) - s), abs(float(F32(p)) - p)
    for c, c0, d in zip(got, py, (ds + dp, ds, dp)):
        assert abs(float(c) - float(c0)) <= d + (_ulp(c) + _ulp(c0)) / 2
    if (s, p) == (3.1, 1.7):
        assert [_ulps(a, b) for a, b in zip(got, py)] == [0, 0, 1]
    if s == 1.1:
        assert _ulps(got[1], py[1]) > 1          # 1 - s is much smaller than s: the rounding of s dominates
    rng = np.random.default_rng(5)
    lg = (rng.standard_normal((3, 4096)) * 5).astype(F32)
    k = keys3(lg[0], lg[1], lg[2], s, p, 1.0).astype(np.float64)
    k0 = G.mix3(torch.from_numpy(lg), s, p).double().numpy()
    terms = np.abs(np.array(py, np.float64))[:, None] * np.abs(lg.astype(np.float64))
    assert np.all(np.abs(k - k0) <= (ds + dp) * np.abs(lg).sum(0) + 5 * 2.0 ** -24 * terms.sum(0))


def test_coefficient_bound_over_random_scales():
    rng = np.random.default_rng(0)
    worst = 0.0
    for s, p in rng.uniform(1, 10, (20000, 2)):
        s, p = float(s), float(p)
        ds, dp = abs(float(F32(s)) - s), abs(float(F32(p)) - p)
        for c, c0, d in zip(coeffs3(s, p), (F32(s + p - 1), F32(1 - s), F32(1 - p)), (ds + dp, ds, dp)):
            bound = d + (_ulp(c) + _ulp(c0)) / 2
            worst = max(worst, abs(float(c) - float(c0)) / bound if bound else 0.0)
    assert worst <= 1.0
    print(f"coefficients from fp32 scales vs Python doubles, 20000 random (s, p): worst |diff| / bound = {worst:.3f}")


@pytest.mark.parametrize("s,p,variant", [(3.1, 1.7, "fp32_sum"), (3.0, 2.0, "right_assoc")])
def test_designed_tie_rows(s, p, variant):
    rows = tie_rows(s, p, variant)
    k = keys3(*rows, s, p, 1.0)
    assert np.all(k == k[0]), "the kernel's keys are not all equal"
    ka = keys3(*rows, s, p, 1.0, **{variant: True})
    assert np.all(ka[0::2] == ka[0]) and np.all(ka[1::2] == ka[1]) and ka[0] != ka[1], "the altered keys do not split"
