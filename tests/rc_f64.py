"""Float64 reference of the gradient reconstruction (es_grad_reconstruct): ``out_p = sum_k w_k table[idx_k + p]``.

TEST INFRASTRUCTURE ONLY.  Nothing here imports the kernel.

* ``rc_layout`` restates the launch plan of ``es_impl_grad_reconstruct`` (reconstruct.cu, ``ES_RC_CTAS_PER_SM`` unset): column
  tiles of 1024, slice chunks of ``k_per_chunk`` (a multiple of 4, at most 1024), and the two refusals.
* ``truth_cols`` / ``truth_device`` give the float64 sum and the per-column mass ``M_p = sum_k |w_k eps_{k,p}|``, slice by slice in
  chunks so that K x P is never held at once.
* ``emulate`` follows the kernel's summation order in numpy float32: every chunk walks its slices in order (zero-weight padding to a
  multiple of 4), then the chunk partials are added in chunk order.  numpy has no ``fmaf``, so each product and each add is
  rounded: the error has the kernel's size, not its bits.  ``emulate(mutation=)`` computes it wrongly on purpose (``MUTATIONS``).
* ``judge`` is the one check the CPU calibration and the GPU test share: the first-order bound of the kernel's order per
  column, and the rms of the error in units of ``U * M_p`` over the columns.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np

U = 2.0 ** -24
TILE = 1024                # RC_TILE_P
MAX_CHUNK = 1024           # RC_MAX_CHUNK
CTAS_PER_SM = 4            # launch bound, ES_RC_CTAS_PER_SM's default
H100_SMS = 132             # H100 SXM5

# rms_p((out_p - truth_p) / (U * M_p)) of a correct kernel.  The largest value of tests/test_gpu_reconstruct_f64.py's problems:
#   es_grad_reconstruct on an NVIDIA H100 80GB HBM3 (700 W power limit), all columns:   0.54   (P = 137 734, K = 8: one chunk)
#   emulate (rounded products and adds, numpy float32, CPU, sampled columns):           0.58   (the same problem)
# RMS_BOUND is about 2x the H100's value.  The largest per-column value on the H100 was 0.42 of its bound (the same problem).
RMS_BOUND = 1.1

MUTATIONS = (
    'drop_first_slice',        # the first slice of the last chunk is skipped
    'drop_last_slice',         # the last real slice of the last chunk is skipped
    'drop_padded_tail',        # a chunk whose slice count is not a multiple of 4 loses the slices after its last group of 4
    'drop_partial',            # one chunk's partial is left out of the final sum
    'double_partial',          # one chunk's partial is added twice
    'tile_shift',              # the second column tile starts one column early (column p >= 1024 reads p - 1)
    'slice_plus_one',          # every slice is read at idx + 1
    'weight_next',             # slice k is scaled by w[k + 1]
    'skip_last_tile',          # the last column tile is never written (left at 0)
)


class Layout(NamedTuple):
    n_tiles: int
    k_per_chunk: int
    n_chunks: int


def rc_layout(P: int, n_idx: int, sm: int) -> Layout:
    """es_impl_grad_reconstruct's grid; ValueError with the kernel's message where it refuses."""
    n_tiles = -(-P // TILE)
    target = max(1, (sm * CTAS_PER_SM) // n_tiles)
    kpc = max(8, -(-n_idx // target))
    kpc = min(MAX_CHUNK, -(-kpc // 4) * 4)
    n_chunks = -(-n_idx // kpc)
    if n_chunks > 65535:
        raise ValueError(f'es_grad_reconstruct: too many slice chunks ({n_chunks})')
    if n_chunks > 1 and n_tiles >= 4000:
        raise ValueError('es_grad_reconstruct: P too large for the ticket array')
    return Layout(n_tiles, kpc, n_chunks)


def chunk_sizes(n_idx: int, lay: Layout):
    return [min(lay.k_per_chunk, n_idx - c * lay.k_per_chunk) for c in range(lay.n_chunks)]


def applicable(mutation: str, P: int, n_idx: int, lay: Layout) -> bool:
    return {'drop_first_slice': True, 'drop_last_slice': True,
            'drop_padded_tail': any(kn % 4 for kn in chunk_sizes(n_idx, lay)),
            'drop_partial': lay.n_chunks > 1, 'double_partial': lay.n_chunks > 1,
            'tile_shift': P > TILE, 'slice_plus_one': True, 'weight_next': n_idx > 1,
            'skip_last_tile': True}[mutation]


# ---------------------------------------------------------------------------------------------- float64 truth
def truth_cols(table: np.ndarray, idx: np.ndarray, w: np.ndarray, cols: np.ndarray, step: int = 2048):
    """(truth, mass) at the columns ``cols``, float64, in slices of ``step``."""
    truth = np.zeros(len(cols))
    mass = np.zeros(len(cols))
    w64 = np.asarray(w, dtype=np.float32).astype(np.float64)
    for s in range(0, len(idx), step):
        e = table[idx[s:s + step, None] + cols[None, :]].astype(np.float64)
        truth += w64[s:s + step] @ e
        mass += np.abs(w64[s:s + step]) @ np.abs(e)
    return truth, mass


def truth_device(table, idx, w, P: int, slice_step: int = 256, col_step: int = 1 << 17):
    """(truth, mass) over all P columns: torch float64 on the tensors' device, in blocks of slices and columns."""
    import torch
    truth = torch.zeros(P, dtype=torch.float64, device=table.device)
    mass = torch.zeros(P, dtype=torch.float64, device=table.device)
    w64 = w.to(torch.float64)
    for c0 in range(0, P, col_step):
        c1 = min(P, c0 + col_step)
        cols = torch.arange(c0, c1, device=table.device)
        for s in range(0, idx.numel(), slice_step):
            e = table[idx[s:s + slice_step, None] + cols[None, :]].to(torch.float64)
            truth[c0:c1] += w64[s:s + slice_step] @ e
            mass[c0:c1] += w64[s:s + slice_step].abs() @ e.abs()
    return truth, mass


# ---------------------------------------------------------------------------------------------- the kernel's order, emulated
def emulate(table: np.ndarray, idx: np.ndarray, w: np.ndarray, P: int, lay: Layout, cols: np.ndarray,
            mutation: Optional[str] = None) -> np.ndarray:
    """float32 ``out`` at ``cols`` in the kernel's order (rounded products), optionally with one modelled bug."""
    f32 = np.float32
    n = len(idx)
    kpc, nch = lay.k_per_chunk, lay.n_chunks
    idx = np.asarray(idx, dtype=np.int64) + (1 if mutation == 'slice_plus_one' else 0)
    w = np.asarray(w, dtype=f32)
    if mutation == 'weight_next':
        w = np.roll(w, -1)
    read = cols.copy()
    if mutation == 'tile_shift':
        read[(cols >= TILE) & (cols < 2 * TILE)] -= 1
    wp = np.zeros(nch * kpc, dtype=f32)
    wp[:n] = w
    sizes = chunk_sizes(n, lay)
    k0 = (nch - 1) * kpc
    if mutation == 'drop_first_slice':
        wp[k0] = 0
    elif mutation == 'drop_last_slice':
        wp[k0 + sizes[-1] - 1] = 0
    elif mutation == 'drop_padded_tail':
        for c, kn in enumerate(sizes):
            if kn % 4:
                wp[c * kpc + kn // 4 * 4:c * kpc + kn] = 0
    ip = np.zeros(nch * kpc, dtype=np.int64)
    ip[:n] = idx
    e = table[ip[:, None] + read[None, :]].reshape(nch, kpc, len(cols))
    wp = wp.reshape(nch, kpc)
    acc = np.zeros((nch, len(cols)), dtype=f32)
    for j in range(kpc):
        acc = acc + (wp[:, j, None] * e[:, j, :])          # float32 x float32 -> rounded, then a rounded add
    if nch == 1:
        out = acc[0].copy()
    else:
        mid = (nch - 1) // 2
        out = np.zeros(len(cols), dtype=f32)
        for c in range(nch):
            if mutation == 'drop_partial' and c == mid:
                continue
            out = out + acc[c]
            if mutation == 'double_partial' and c == mid:
                out = out + acc[c]
    if mutation == 'skip_last_tile':
        out[cols >= (lay.n_tiles - 1) * TILE] = 0
    return out


# ---------------------------------------------------------------------------------------------- the check
def judge(out, truth, mass, lay: Layout):
    """(worst, rms): the largest |out - truth| over its first-order bound (k_per_chunk + n_chunks) U M_p, and
    rms_p(|out - truth| / (U M_p)).  A column of zero mass must be exact (else it counts as infinitely wrong)."""
    d = np.abs(np.asarray(out, dtype=np.float64) - truth)
    with np.errstate(divide='ignore', invalid='ignore'):
        unit = np.where(mass > 0, d / (U * mass), np.where(d > 0, np.inf, 0.0))
    worst = float(np.max(unit)) / (lay.k_per_chunk + lay.n_chunks)
    rms = float(np.sqrt(np.mean(unit ** 2)))
    return worst, rms


def passes(worst: float, rms: float) -> bool:
    return worst <= 1.0 and rms <= RMS_BOUND


def margin(worst: float, rms: float) -> float:
    """How far a result is outside the checks: the larger of worst / 1 and rms / RMS_BOUND."""
    return max(worst, rms / RMS_BOUND)
