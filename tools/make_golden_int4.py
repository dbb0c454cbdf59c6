"""Regenerate tests/golden/int4_quant.npz from the reference implementation's own int4 group quantiser.

    python tools/make_golden_int4.py /path/to/metavoice-src

Runs ``fam.llm.fast_quantize.group_quantize_tensor(w, 4, 128)`` and ``group_dequantize_tensor_from_qparams`` (both plain
torch on the CPU) on seeded bf16 matrices: slices of the production shapes (K = 256, 2048, 5632) and one matrix of edge-case
groups.  Stored per case: the bf16 input (as uint16 bits), q (uint8), scales / zeros (uint16 bf16 bits, [M, K/128]) and the
reference's dequantised weight (uint16 bf16 bits)."""
import sys

import numpy as np
import torch


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def edge_matrix() -> torch.Tensor:
    """8 rows x 2 groups; each group exercises one edge of the quantiser."""
    g = torch.Generator().manual_seed(5)
    rows = []
    rnd = lambda scale: torch.randn(128, generator=g) * scale                                   # noqa: E731
    groups = [
        torch.full((128,), 0.0371),                                    # constant: range 0 -> clamped to 1e-6
        torch.zeros(128),                                              # all zero
        0.25 + rnd(1e-8),                                              # range below the 1e-6 clamp
        torch.cat([rnd(0.01)[:127], torch.tensor([3.5])]),             # one outlier
        -(rnd(0.05).abs() + 0.01),                                     # negative only
        rnd(1.0) * 4e37,                                               # near the top of the bf16 range (max - min stays finite)
        rnd(1.0) * 1e-37,                                              # near the bottom of the normal bf16 range
        torch.cat([torch.full((64,), -2.0), torch.full((64,), 2.0)]),  # two values: exact grid points
        rnd(0.02),
        torch.linspace(-1, 1, 128),
        rnd(3.0),
        torch.full((128,), -7.0),
        rnd(1e-3) + 100.0,
        torch.cat([torch.tensor([-1e30]), rnd(1.0)[1:]]),
        rnd(0.5).clamp(min=0),
        torch.arange(128.0) / 8,
    ]
    for i in range(0, len(groups), 2):
        rows.append(torch.cat([groups[i], groups[i + 1]]))
    return torch.stack(rows).to(torch.bfloat16)


def main(ref_root: str) -> None:
    sys.path.insert(0, ref_root)
    from fam.llm.fast_quantize import group_dequantize_tensor_from_qparams, group_quantize_tensor

    g = torch.Generator().manual_seed(2024)
    cases = {
        "k256": (torch.randn(64, 256, generator=g) * 0.05).to(torch.bfloat16),    # speaker_cond_pos slice
        "k2048": (torch.randn(48, 2048, generator=g) * 0.02).to(torch.bfloat16),  # wqkv / wo / w1 / w3 slice
        "k5632": (torch.randn(16, 5632, generator=g) * 0.02).to(torch.bfloat16),  # w2 slice
        "edge": edge_matrix(),
    }
    out = {}
    for name, w in cases.items():
        w_int32, sz = group_quantize_tensor(w, 4, 128)            # sz: [K/128, M, 2] (scale, zero)
        scales = sz[..., 0].t().contiguous()
        zeros = sz[..., 1].t().contiguous()
        w_dq = group_dequantize_tensor_from_qparams(w_int32, scales, zeros, 4, 128)
        assert w_dq.dtype == torch.bfloat16
        out[f"{name}_w"] = _bits(w)
        out[f"{name}_q"] = w_int32.to(torch.uint8).numpy()
        out[f"{name}_scales"] = _bits(scales)
        out[f"{name}_zeros"] = _bits(zeros)
        out[f"{name}_deq"] = _bits(w_dq)
    np.savez_compressed("tests/golden/int4_quant.npz", **out)
    print("wrote tests/golden/int4_quant.npz:", ", ".join(f"{k}{list(v.shape)}" for k, v in out.items()))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else ".")
