"""FP8 weights without a GPU: the quantizer rule of tests/fp8_oracle.py (the reference the GPU kernels are compared with),
the exactness of bf16(Q * 2^e) that makes an fp8 engine bit-identical to a bf16 engine on the dequantized weights, and the
`litellm_params.quantization` config key."""
import numpy as np
import pytest
import torch

import fp8_oracle as ref


def _e4m3_values():
    """Every finite e4m3 value (codes 0x00..0x7e and their negatives), as float64."""
    codes = torch.arange(256, dtype=torch.uint8)
    v = codes.view(torch.float8_e4m3fn).double()
    return v[torch.isfinite(v)]


def _numpy_rne_e4m3(x: np.ndarray) -> np.ndarray:
    """Independent round-to-nearest-even onto the e4m3 grid (|x| <= 448): the grid spacing of a binade is 2^(E - 3) for
    E >= -6 and 2^-9 below (subnormals)."""
    ax = np.abs(x)
    E = np.floor(np.log2(np.where(ax > 0, ax, 1.0)))
    step = np.exp2(np.maximum(E, -6) - 3)
    return np.sign(x) * np.round(ax / step) * step        # np.round: halves to even


def test_torch_e4m3_conversion_is_rne_with_subnormals():
    pos = np.sort(_e4m3_values().numpy()[_e4m3_values().numpy() > 0])
    assert pos[0] == 2.0 ** -9 and pos[-1] == 448.0 and len(pos) == 126
    mids = ((pos[:-1] + pos[1:]) / 2).astype(np.float32)       # fp32 probes: the quantizer converts from fp32
    probes = np.concatenate([pos.astype(np.float32), mids, np.nextafter(mids, np.float32(0)),
                             np.nextafter(mids, np.float32(np.inf)), np.float32([2.0 ** -10, 2.0 ** -11, 3 * 2.0 ** -11])])
    probes = np.concatenate([probes, -probes])
    got = torch.from_numpy(probes).to(torch.float8_e4m3fn).double().numpy()
    probes = probes.astype(np.float64)
    np.testing.assert_array_equal(got, _numpy_rne_e4m3(probes))
    # ties go to the even code: the midpoint of codes 1 and 2 (subnormals) rounds to 2, of 2 and 3 to 2
    t = torch.tensor([1.5 * 2.0 ** -9, 2.5 * 2.0 ** -9]).to(torch.float8_e4m3fn)
    assert t.view(torch.uint8).tolist() == [2, 2]


@pytest.mark.parametrize("k", [-120, -117, -60, -9, 0, 1, 7, 60, 119])   # 448 * 2^119: the largest bound a bf16 reaches
def test_exponent_is_the_smallest_with_amax_within_448_times_2e(k):
    w = torch.zeros(4, 64, dtype=torch.float64)
    w[0, 3] = 448.0 * 2.0 ** k                                             # exactly at the bound: e = k
    w[1, 5] = -450.0 * 2.0 ** k                                            # just above: the next bf16 after 448
    w[2, 7] = 448.0 * 2.0 ** (k - 1)                                       # e = k - 1
    w[3, 9] = 2.0 ** k                                                      # a power of two: 1 * 2^k <= 448 * 2^(k - 8)
    wb = w.bfloat16()
    e = ref.row_exponents(wb)
    clamp = lambda v: max(ref.E_MIN, min(ref.E_MAX, v))
    assert e.tolist() == [clamp(k), clamp(k + 1), clamp(k - 1), clamp(k - 8)]
    for n in range(4):
        a = wb[n].double().abs().max().item()
        en = e[n].item()
        if ref.E_MIN < en < ref.E_MAX:
            assert a <= 448 * 2.0 ** en and a > 448 * 2.0 ** (en - 1)


def test_zero_rows_clamped_rows_and_subnormal_outputs():
    w = torch.zeros(3, 32, dtype=torch.float64)
    w[1] = 2.0 ** -130 * torch.arange(1, 33)                                # amax 2^-125: below the clamp, e = -117
    w[2, 0], w[2, 1], w[2, 2] = 448.0, 2.0 ** -8, 3 * 2.0 ** -11            # e = 0: two subnormal outputs
    wb = w.bfloat16()
    q, s = ref.quantize(wb)
    assert s.tolist() == [1.0, 2.0 ** -117, 1.0]
    assert q[0].double().abs().sum() == 0
    # row 1: values 2^-13 .. 2^-8 after scaling: the small ones round to 0 or to e4m3 subnormals, none saturates
    assert torch.isfinite(q[1].double()).all() and q[1].double().abs().max() <= 448
    assert q[2, 1].double() == 2.0 ** -8                                    # exact subnormal
    assert q[2, 2].double() == 2.0 ** -9                                    # 0.75 steps of 2^-9 round up to one
    d = ref.dequantize(q, s)
    assert torch.equal(d.double(), q.double() * s.double()[:, None])


def test_dequantized_value_is_exact_for_every_e4m3_value_and_exponent():
    v = _e4m3_values()                                                      # 253 finite values (with both zeros)
    e = torch.arange(ref.E_MIN, ref.E_MAX + 1, dtype=torch.float64)
    prod = v[:, None] * torch.exp2(e)[None, :]
    # Products beyond the bf16 range need a row amax within 2^-4 of bf16's largest value (its e4m3 code rounds up past
    # 2^128); every other product is exact.
    bf16_max = torch.finfo(torch.bfloat16).max
    prod = prod[prod.abs() <= bf16_max]
    assert torch.equal(prod.bfloat16().double(), prod)
    # and fp32 holds every product as a normal number (the conversion path multiplies in fp32)
    nz = prod[prod != 0].abs()
    assert nz.min() >= 2.0 ** -126 and torch.equal(prod.float().double(), prod)


def test_quantize_round_trip_error_is_bounded_by_half_an_e4m3_step():
    g = torch.Generator().manual_seed(3)
    w = (torch.randn(64, 256, generator=g) * 0.02).bfloat16()
    q, s = ref.quantize(w)
    d = ref.dequantize(q, s).double()
    err = (d - w.double()).abs()
    # relative step of e4m3 normals is 2^-3; subnormal step 2^-9 * s
    bound = torch.maximum(w.double().abs() * 2.0 ** -4, 2.0 ** -10 * s.double()[:, None])
    assert (err <= bound * (1 + 1e-12)).all()


# ---- config --------------------------------------------------------------------------------------------------------------
def _cfg(*lps):
    from rr_b200.config import build_config
    return build_config([{"model_name": "m", "litellm_params": dict(model="b200/tiny", **lp)} for lp in lps])


@pytest.mark.parametrize("value", [None, "fp8"])
def test_quantization_accepted_values(value):
    lp = {} if value is None else {"quantization": value}
    assert _cfg(lp).deployments[0].quantization == value
    assert _cfg({"quantization": None}).deployments[0].quantization is None


@pytest.mark.parametrize("value", ["FP8", "int8", "bf16", "fp8_e4m3", 8, True, ["fp8"]])
def test_quantization_other_values_refused(value):
    with pytest.raises(ValueError, match="quantization"):
        _cfg({"quantization": value})


def test_quantization_must_agree_on_a_shared_gpu():
    with pytest.raises(ValueError, match="disagree on litellm_params.quantization"):
        _cfg({"quantization": "fp8", "gpu": 0}, {"gpu": 0})
    cfg = _cfg({"quantization": "fp8", "gpu": 0}, {"gpu": 1})
    assert [d.quantization for d in cfg.deployments] == ["fp8", None]


def test_fp8_config_file_loads():
    import os
    from rr_b200.config import load_config
    cfg = load_config(os.path.join(os.path.dirname(__file__), "..", "config", "fp8.yaml"))
    assert [d.quantization for d in cfg.deployments] == ["fp8"]


def test_stub_backends_validate_and_ignore_quantization():
    from rr_b200.server import build_backends
    cfg = _cfg({"quantization": "fp8"})
    assert len(build_backends(cfg, stub=True)) == 1
