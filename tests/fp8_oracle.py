"""CPU ORACLE of the e4m3 corpus storage (FLMR_CORPUS_FP8) — TEST INFRASTRUCTURE ONLY.

The scan of an fp8 corpus computes MaxSim of e4m3(Q) against e4m3(D) with fp32 accumulation: both operands
rounded to nearest even (saturating at +-448, no scale), then the exact MaxSim of ``oracle/maxsim_oracle.py``.
"""
from __future__ import annotations

import numpy as np

from oracle import maxsim_oracle as O

E4M3_MAX = 448.0


def e4m3_round(x: np.ndarray) -> np.ndarray:
    """fp32 -> float8 e4m3fn -> fp32, round to nearest even, saturated (what ``cvt.rn.satfinite.e4m3x2.f32`` does;
    torch's ``.to(torch.float8_e4m3fn)`` agrees inside +-448).  e4m3: 3 mantissa bits, normals from 2^-6,
    subnormals in steps of 2^-9."""
    x = np.asarray(x, dtype=np.float32)
    a = np.abs(x).astype(np.float64)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -9)))
    step = 2.0 ** (np.maximum(e, -6.0) - 3.0)             # spacing of the binade (subnormal: 2^-9)
    r = np.minimum(np.round(a / step) * step, E4M3_MAX)   # np.round: half to even
    return np.where(x < 0, -r, r).astype(np.float32)


def maxsim_scores_fp8(Q: np.ndarray, D_packed: np.ndarray, doclens: np.ndarray, relu: bool = False) -> np.ndarray:
    """``out[b, p] = sum_i max_{j<len_p} <e4m3(Q[b,i]), e4m3(D_p[j])>`` (fp32)."""
    return O.maxsim_scores(e4m3_round(Q), e4m3_round(D_packed), doclens, relu=relu)
