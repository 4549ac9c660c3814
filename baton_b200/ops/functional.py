"""Functional wrappers over the sm_90a kernels (shape logic + dispatch).

Conventions
-----------
* activations are bf16, row-major; images are NHWC (``[N, H, W, C]``);
* a GEMM operand is a 2-D tensor with unit inner stride; ``*_mn=False`` means the
  tensor is ``[rows, K]`` (K-major), ``*_mn=True`` means it is ``[K, rows]``
  (MN-major) -- so forward / dgrad / wgrad need no transposes;
* kernels that produce parameter gradients *accumulate* into fp32 buffers (the
  flat gradient arena), the fused SGD step zeroes them again.
"""
from __future__ import annotations

import collections
import functools
from typing import List, Optional, Sequence, Tuple

import torch

from ._ext import load

BF16 = torch.bfloat16
NUM_SMS = 132          # H100 SXM: wave counts of the dispatch heuristics below


def _pitch(t: torch.Tensor) -> int:
    assert t.dim() == 2 and (t.stride(1) == 1 or t.shape[1] == 1), "GEMM operand must have unit inner stride"
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def _tma_ok(t: torch.Tensor) -> bool:
    return t.dtype == BF16 and _pitch(t) % 8 == 0 and t.data_ptr() % 16 == 0


def pick_bn(M: int, N: int) -> int:
    """Widest N tile the GEMM kernels instantiate (128) when it still yields enough CTAs; 64 for small problems.
    The split-K heuristics below count output tiles with this width, so it must be the width that actually runs."""
    m_tiles = (M + 127) // 128
    if N >= 128 and m_tiles * ((N + 127) // 128) >= NUM_SMS:
        return 128
    if N > 128 and m_tiles * ((N + 127) // 128) >= NUM_SMS // 2:
        return 128
    return 64


_WGRAD_MAX_CTAS = 64        # CTAs of one split-K weight-gradient launch (see pick_split_k)
_CLUSTER_MIN_KT = 4         # k tiles every CTA of a split-K cluster must keep (see pick_cluster_k)


def pick_split_k(M: int, N: int, K: int, bn: int) -> int:
    """Atomic split-K factor of a weight-gradient GEMM.  ``_WGRAD_MAX_CTAS`` caps the CTAs of one launch: these
    GEMMs run as a parallel graph branch beside the dgrad / BatchNorm chain and should leave SMs to it."""
    tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
    k_tiles = (K + 63) // 64
    if tiles >= NUM_SMS // 2 or k_tiles < 8:
        return 1
    return max(1, min(k_tiles // 4, max(1, _WGRAD_MAX_CTAS // tiles)))


def pick_cluster_k(M: int, N: int, K: int, bn: int) -> int:
    """Cluster split-K factor (1, 2, 4 or 8) for GEMMs with few output tiles and a long K."""
    tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
    k_tiles = (K + 63) // 64
    if k_tiles < 16:     # short main loops gain nothing from splitting
        return 1
    best = 1
    for s in (2, 4, 8):
        # clusters of 8 only pay off while they cover at most ~half the SMs
        # (placement needs 8 free SMs inside one GPC); clusters of <= 4 are fine up to a full wave
        cap = NUM_SMS // 2 if s == 8 else 128
        if tiles * s <= cap and k_tiles >= _CLUSTER_MIN_KT * s:
            best = s
    return best


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = BF16, bias: Optional[torch.Tensor] = None,
         act: int = 0, accumulate: bool = False, alpha: float = 1.0, split_k: Optional[int] = None,
         n_valid: Optional[int] = None, flags: Optional[torch.Tensor] = None, flag_epoch: int = 0,
         flag_elem_off: int = 0, flag_tile_elems: int = 0, flag_bias_off: int = -1, force_bn: int = 0,
         force_simt: bool = False, col_stats: Optional[torch.Tensor] = None,
         flag_epoch_word: Optional[torch.Tensor] = None, sgd: Optional[dict] = None,
         affine: Optional[dict] = None) -> Optional[torch.Tensor]:
    """``out[M,N] = act(alpha * A @ B^T + bias)`` on the tensor cores (wgmma).

    ``n_valid`` limits the written columns (used when B carries zero K-padding
    rows, e.g. the wgrad of a layer whose K was padded to a multiple of 8).

    ``col_stats`` (fp32 ``[2N]``): the epilogue also accumulates the per-column sum and sum of squares of the
    bf16 output into it -- the BatchNorm batch statistics of a convolution, without a second pass over the
    activation.  Only legal where :func:`gemm_stats_fusable` says so (single-pass tensor-core GEMM).

    ``sgd`` (see :func:`sgd_epilogue_args`): on a weight-gradient GEMM (``accumulate`` into fp32 ``out``, MN-major
    operands) apply the SGD step to the parameters in the epilogue instead of accumulating the gradient into ``out``.
    Returns ``None`` when this GEMM cannot (split-K, persistent kernel...): nothing was written, accumulate instead.

    ``affine`` (see :func:`affine_epilogue_args`): eval-mode BatchNorm in the epilogue of a bf16 forward GEMM,
    ``out = relu?(A @ B^T * scale + shift + residual)``.  Returns ``None`` when this GEMM cannot apply it: nothing was
    written, run the GEMM and ``bn_apply`` instead."""
    C = load()
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    assert K == Kb, "GEMM reduction dims differ: {} vs {}".format(K, Kb)
    if n_valid is not None:
        N = min(N, n_valid)
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=a.device)
        if accumulate:
            out.zero_()
    ldd = out.stride(0) if out.dim() == 2 else N
    lda, ldb = _pitch(a), _pitch(b)
    use_simt = force_simt or not (_tma_ok(a) and _tma_ok(b))
    if use_simt and (sgd is not None or affine is not None):
        return None
    if use_simt:
        assert col_stats is None, "fused column statistics need the tensor-core path"
        C.gemm(a, b, out, bias, M, N, K, lda, ldb, ldd, a_mn, b_mn, act, 1, accumulate, alpha, None, 0, 0, 0, -1, 0,
               True, None, None, None, None, None, None, False, None, None, None, None, None, None, False)
        return out
    bn = force_bn or pick_bn(M, N)
    if col_stats is not None:
        assert not accumulate and bias is None and act == 0 and alpha == 1.0
    if split_k is None:
        if accumulate and out.dtype == torch.float32:
            split_k = pick_split_k(M, N, K, bn)          # atomic split-K straight into the gradient arena
        else:
            split_k = -pick_cluster_k(M, N, K, bn)       # cluster split-K, DSMEM reduce (negative = cluster)
            if split_k == -1:
                split_k = 1
    if split_k > 1:
        assert out.dtype == torch.float32 and bias is None and act == 0
    if sgd is not None and split_k != 1:
        return None                 # the optimizer epilogue needs every tile's complete gradient in one CTA
    if affine is not None and split_k > 1:
        return None                 # atomic split-K partials cannot take a per-element epilogue
    sg, af = sgd or {}, affine or {}
    if not C.gemm(a, b, out, bias, M, N, K, lda, ldb, ldd, a_mn, b_mn, act, split_k, accumulate, alpha, flags, flag_epoch,
                  flag_elem_off, flag_tile_elems, flag_bias_off, bn, False, col_stats, flag_epoch_word, sg.get("theta"),
                  sg.get("theta_bf16"), sg.get("momentum"), sg.get("hyper"), bool(sg.get("nesterov", False)),
                  sg.get("anchor"), sg.get("corr"), sg.get("adam_v"), af.get("scale"), af.get("shift"), af.get("residual"), bool(af.get("relu", False))):
        return None
    return out


def lora_down(x: torch.Tensor, w: torch.Tensor, *, T: int, rs: int, kt: int, xoff: Sequence[int], w_ts: int, wsj: int,
              wsk: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LoRA down projection ``U[m, t rs + j] = bf16(sum_k x[m, xoff[t] + k] * w[t w_ts + j wsj + k wsk])`` for ``T``
    slices, ``k < kt`` (csrc/lora.cu): ``U = X A^T`` in the forward, ``V = dY' B`` per targeted slice in the backward.
    Returns ``[M, T rs]`` bf16 (``out`` when given)."""
    M = x.shape[0]
    u = torch.empty((M, T * rs), dtype=BF16, device=x.device) if out is None else out
    load().lora_down(x, _pitch(x), w, w_ts, wsj, wsk, u, _pitch(u), M, T, rs, kt, list(xoff))
    return u


def gemm_lora(a: torch.Tensor, b: torch.Tensor, lora: dict, *, b_mn: bool = False, bias: Optional[torch.Tensor] = None,
              act: int = 0, out_dtype: torch.dtype = BF16, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``act(A @ B^T + s T + bias)`` with the rank term ``T`` of ``lora`` in the GEMM epilogue (``B200LoraEpilogue`` in
    csrc/launch.h): keys ``u`` (bf16 ``[M, R]``), ``f``, ``fs_n``, ``fs_j``, ``rs``, ``ds``, ``slot`` (three entries) and
    ``s``.  ``A`` is K-major ``[M, K]``; ``B`` is ``[N, K]``, or ``[K, N]`` with ``b_mn``."""
    M, K = a.shape
    N = b.shape[1] if b_mn else b.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    u = lora["u"]
    load().gemm_lora(a, b, out, bias, M, N, K, _pitch(a), _pitch(b), _pitch(out), False, b_mn, act, 1.0, u, _pitch(u), lora["f"],
                     lora["fs_n"], lora["fs_j"], u.shape[1], lora["rs"], lora["ds"], list(lora["slot"]), lora["s"])
    return out


def lora_grad_(l: torch.Tensor, q: torch.Tensor, out: torch.Tensor, *, NA: int, NB: int, lo: Sequence[int],
               qo: Sequence[int], osa: int, osb: int, out_ts: int, s: float) -> None:
    """Adapter gradient ``out[t out_ts + a osa + b osb] += s * sum_m l[m, lo[t] + a] * q[m, qo[t] + b]`` (csrc/lora.cu):
    ``dA = s V^T X`` and ``dB = s dY'^T U``.  A fixed split over M, summed in a fixed order: the bits do not depend on
    the device, the run or graph capture."""
    C = load()
    M, T = l.shape[0], len(lo)
    splits = -(-M // C.LORA_SPLIT_ROWS)
    work = torch.empty(T * splits * NA * NB, dtype=torch.float32, device=l.device)
    C.lora_grad(l, _pitch(l), q, _pitch(q), out, osa, osb, out_ts, M, NA, NB, T, list(lo), list(qo), s, work)


def affine_epilogue_args(table: torch.Tensor, offset: int, channels: int, relu: bool,
                         residual: Optional[torch.Tensor] = None) -> dict:
    """``affine=`` argument of :func:`gemm` / :func:`conv_igemm_fwd` for the BatchNorm whose eval scale / shift
    :func:`bn_fold_eval` wrote at ``offset`` of ``table``; ``residual``: optional bf16 ``[rows, channels]`` (or NHWC)
    tensor added before the ReLU."""
    return {"scale": table[offset: offset + channels], "shift": table[offset + channels: offset + 2 * channels],
            "relu": relu, "residual": residual}


def bn_fold_eval(arena: torch.Tensor, table: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Eval-mode scale / shift of every BatchNorm of ``table`` (int64 ``[n_bn, 7]``: element offsets of gamma, beta,
    running_mean, running_var in the fp32 ``arena``, output offset, C, eps as float32 bits) into ``out``, one launch:
    ``scale = gamma * rsqrt(var + eps)``, ``shift = beta - mean * gamma * rsqrt(var + eps)`` -- ``bn_apply``'s eval
    arithmetic."""
    load().bn_fold_eval(arena, table, out)
    return out


def gemm_stats_fusable(M: int, N: int, K: int) -> bool:
    """Can :func:`gemm` take column statistics of this problem in its epilogue?  Every bf16-output tensor-core
    path can: single-pass tiles do it from the staged accumulator rows (butterfly column sums), cluster split-K in the DSMEM
    reduction; only operands that fall back to the SIMT kernel (pitch not a multiple of 8) cannot."""
    return K % 8 == 0


# ---------------------------------------------------------------------------- elementwise / optimizer
def fused_sgd(w: torch.Tensor, g: torch.Tensor, hyper: torch.Tensor, momentum_buf: Optional[torch.Tensor] = None,
              w_bf16: Optional[torch.Tensor] = None, zero_grad: bool = True, nesterov: bool = False,
              pack: Optional[dict] = None, prox_anchor: Optional[torch.Tensor] = None,
              corr: Optional[torch.Tensor] = None, adam_v: Optional[torch.Tensor] = None, clip: bool = False) -> None:
    """One kernel over the whole flat arena (reference: ``optimizer.step()``, demo.py:47).

    ``clip`` (gradient-norm clipping): the gradient is multiplied by the coefficient :func:`grad_norm_clip` wrote, as it
    is loaded and before any other term -- ``hyper[SGD_HYPER_CLIP]`` (``hyper`` then holds 6 floats) or, with AdamW,
    ``hyper[ADAMW_ROW_CLIP]`` of the step's row.

    ``adam_v`` (AdamW, exclusive with ``prox_anchor`` and ``corr``): fp32 second moment indexed like ``w``; the step is
    then AdamW's, ``momentum_buf`` (required) is the first moment and ``hyper`` the step's row of :func:`adamw_rows`.

    ``prox_anchor`` (FedProx): fp32 buffer indexed like ``w`` (the global model the round started from); the step adds
    ``hyper[4] * (w - prox_anchor)`` to the gradient, so ``hyper`` then holds 5 floats
    ``[lr, momentum, weight_decay, dampening, prox_mu]``.  ``None``: no proximal term, ``hyper[4]`` is never read.

    ``corr`` (SCAFFOLD, exclusive with ``prox_anchor``): fp32 buffer indexed like ``w`` holding ``c - c_i``; the step
    adds it to the gradient after weight decay.

    ``pack`` (SURVEY K4, "emits the upload copy"): ``{"wire_slot": int64[1] device word holding the wire address,
    "global_w": fp32 global copy or None, "scale": fp32[1] device scalar or None, "n_pack": elements to pack
    (parameters + float buffers), "wire_fp32": bool}`` -- the step also writes this client's wire copy for the
    round-end collective while the new weights are in registers."""
    pk = pack or {}
    load().fused_sgd(w, g, momentum_buf, w_bf16, hyper, zero_grad, nesterov, pk.get("wire_slot"),
                     pk.get("global_w"), pk.get("scale"), int(pk.get("n_pack", 0)), bool(pk.get("wire_fp32", False)),
                     prox_anchor, corr, adam_v, bool(clip))


ADAMW_ROW = 12         # floats per AdamW step row (csrc/sgd.cuh: ADAMW_ROW / AdamHyper)
SGD_HYPER_CLIP = 5     # the clip coefficient's float in the SGD hyper-parameters (csrc/sgd.cuh)
ADAMW_ROW_CLIP = 9     # ... and in an AdamW step row


def grad_norm_clip(g: torch.Tensor, max_norm: torch.Tensor, work: torch.Tensor, norm_out: torch.Tensor,
                   coef_out: torch.Tensor) -> None:
    """``clip_grad_norm_``'s norm and coefficient on the device: ``norm_out[0] = ||g||`` (fp32, accumulated in fp64 with
    a fixed grid and summation order: the same bits on every launch) and ``coef_out[0] = min(max_norm[0] / (norm +
    1e-6), 1)`` rounded as torch rounds it from the fp32 norm.  ``max_norm``: fp32 device scalar.  ``work``: int64
    ``[GRAD_NORM_WORK_WORDS]`` of zeros, reusable by launches on the same stream; its last word holds the fp64 sum of
    squares afterwards."""
    load().grad_norm_clip(g, max_norm, work, norm_out, coef_out)


def adamw_rows(lr: float, betas: Tuple[float, float], eps: float, weight_decay: float, t0: int, count: int,
               first: bool = True) -> torch.Tensor:
    """fp32 ``[count, ADAMW_ROW]`` AdamW coefficients of local steps ``t0 .. t0 + count - 1`` (``t`` counts from 1),
    computed in fp64 and rounded once: ``{1 - lr*wd, b1, 1 - b1, b2, 1 - b2, eps, lr / (1 - b1^t),
    1 / sqrt(1 - b2^t), t == 1}`` -- the bias corrections of ``torch.optim.AdamW``.  ``first=False`` never marks a
    row as the first step."""
    b1, b2 = float(betas[0]), float(betas[1])
    lr, eps, wd = float(lr), float(eps), float(weight_decay)
    rows = torch.zeros(count, ADAMW_ROW, dtype=torch.float64)
    t = torch.arange(t0, t0 + count, dtype=torch.float64)
    rows[:, 0] = 1.0 - lr * wd
    rows[:, 1], rows[:, 2], rows[:, 3], rows[:, 4], rows[:, 5] = b1, 1.0 - b1, b2, 1.0 - b2, eps
    rows[:, 6] = lr / (1.0 - torch.pow(torch.tensor(b1, dtype=torch.float64), t))
    rows[:, 7] = 1.0 / torch.sqrt(1.0 - torch.pow(torch.tensor(b2, dtype=torch.float64), t))
    rows[:, 8] = ((t == 1) & first).to(torch.float64)
    return rows.to(torch.float32)


def sgd_epilogue_args(theta: torch.Tensor, grad: torch.Tensor, grad_view: torch.Tensor, hyper: torch.Tensor,
                      momentum: Optional[torch.Tensor] = None, theta_bf16: Optional[torch.Tensor] = None,
                      nesterov: bool = False, anchor: Optional[torch.Tensor] = None,
                      corr: Optional[torch.Tensor] = None, adam_v: Optional[torch.Tensor] = None) -> dict:
    """``sgd=`` argument of a weight-gradient GEMM whose output ``grad_view`` is a view of the flat gradient ``grad``:
    the parameter, bf16 shadow, momentum, FedProx anchor, SCAFFOLD correction and AdamW second-moment buffers (same
    offsets as ``grad``) from the element ``grad_view[0, 0]`` on.  With an ``anchor`` the step is the one of
    :func:`fused_sgd` with ``prox_anchor``, with a ``corr`` the one with ``corr``, with an ``adam_v`` AdamW's."""
    off = (grad_view.data_ptr() - grad.data_ptr()) // grad.element_size()
    assert 0 <= off < grad.numel(), "the GEMM output is not a view of the gradient arena"
    return {"theta": theta[off:], "theta_bf16": theta_bf16[off:] if theta_bf16 is not None else None,
            "momentum": momentum[off:] if momentum is not None else None, "hyper": hyper, "nesterov": nesterov,
            "anchor": anchor[off:] if anchor is not None else None, "corr": corr[off:] if corr is not None else None,
            "adam_v": adam_v[off:] if adam_v is not None else None}


SGD_CHUNK = 8192       # arena elements per chunk of the leftover optimizer pass (one CTA iteration each)


def sgd_segments(n: int, fused: Sequence[Tuple[int, int, int, int]], nograd: Sequence[Tuple[int, int]],
                 chunk: int = SGD_CHUNK) -> List[Tuple[int, int, int]]:
    """Chunk table of the leftover optimizer pass of a step whose weight-gradient GEMMs applied SGD in their epilogue.

    ``fused``: ``(offset, rows, cols, ld)`` element blocks the epilogues updated (row ``r`` covers
    ``[offset + r * ld, offset + r * ld + cols)``); ``nograd``: ``(offset, length)`` parameter ranges whose gradient is
    identically zero outside the fused blocks.  Returns ``(offset, length, kind)`` chunks of at most ``chunk`` elements
    that cover ``[0, n)`` minus the fused blocks exactly once, in offset order; kind 1 inside a ``nograd`` range, else
    0."""
    pieces = sorted((o + r * ld, o + r * ld + cols) for o, rows, cols, ld in fused for r in range(rows))
    free, pos = [], 0
    for s, e in pieces:
        if s < pos or e > n:
            raise ValueError("fused blocks overlap or leave the arena: [{}, {})".format(s, e))
        if s > pos:
            free.append((pos, s))
        pos = e
    if pos < n:
        free.append((pos, n))
    ng = sorted((o, o + l) for o, l in nograd)
    out = []
    for s, e in free:
        cuts = sorted({s, e} | {b for r in ng for b in r if s < b < e})
        for a, b in zip(cuts, cuts[1:]):
            kind = 1 if any(lo <= a and b <= hi for lo, hi in ng) else 0
            out.extend((c, min(chunk, b - c), kind) for c in range(a, b, chunk))
    return out


def fused_sgd_segments(w: torch.Tensor, g: torch.Tensor, hyper: torch.Tensor, segments: torch.Tensor,
                       momentum_buf: Optional[torch.Tensor] = None, w_bf16: Optional[torch.Tensor] = None,
                       nesterov: bool = False, prox_anchor: Optional[torch.Tensor] = None,
                       corr: Optional[torch.Tensor] = None, adam_v: Optional[torch.Tensor] = None,
                       clip: bool = False) -> None:
    """The step of :func:`fused_sgd` over the arena chunks of ``segments`` (device int64 ``[S, 3]`` from
    :func:`sgd_segments`); chunks of kind 1 never read the gradient.  ``prox_anchor``, ``corr``, ``adam_v`` and
    ``clip`` as in :func:`fused_sgd`; a kind-1 element without a momentum buffer (or with AdamW) is then written only
    where the step changes it."""
    load().fused_sgd_segments(w, g, momentum_buf, w_bf16, segments, hyper, nesterov, prox_anchor, corr, adam_v,
                              bool(clip))


def scaffold_corr(corr: torch.Tensor, c: torch.Tensor, c_i: torch.Tensor) -> None:
    """SCAFFOLD: ``corr = c - c_i`` over ``corr.numel()`` parameters, the correction client ``i`` trains with."""
    load().scaffold_corr(corr, c, c_i)


def scaffold_dc(up: torch.Tensor, c_i: torch.Tensor, c: torch.Tensor, global_w: torch.Tensor, theta: torch.Tensor,
                inv_k_eta: float, *, first: bool) -> None:
    """SCAFFOLD after client ``i`` trained ``K`` steps at learning rate ``eta`` (option II): ``dc = (global_w - theta)
    * inv_k_eta - c`` with ``inv_k_eta = 1 / (K eta)``; ``c_i += dc``; ``up = dc`` (``first``) or ``up += dc``.  Over
    ``up.numel()`` parameters."""
    load().scaffold_dc(up, c_i, c, global_w, theta, float(inv_k_eta), bool(first))


def weighted_sum_(dst: torch.Tensor, srcs: Sequence[torch.Tensor], weights: Sequence[float]) -> torch.Tensor:
    """``dst = sum_k weights[k] * srcs[k]`` in one pass (manager-side FedAvg, manager.py:124-126)."""
    C = load()
    flat_dst = dst.view(-1) if dst.is_contiguous() else None
    if flat_dst is None or dst.dtype not in (torch.float32, BF16) or len(srcs) > C.MAX_RANKS:
        acc = torch.zeros_like(dst, dtype=torch.float32)
        for s, w in zip(srcs, weights):
            acc.add_(s.to(device=dst.device, dtype=torch.float32), alpha=float(w))
        dst.copy_(acc.to(dst.dtype))
        return dst
    ss = [s.to(device=dst.device, dtype=dst.dtype).contiguous().view(-1) for s in srcs]
    C.weighted_sum(flat_dst, ss, [float(w) for w in weights])
    return dst


def fold_client(acc: torch.Tensor, theta: torch.Tensor, global_w: torch.Tensor, nk: float, *, first: bool = False,
                reset: bool = False, w_bf16: Optional[torch.Tensor] = None, momentum: Optional[torch.Tensor] = None) -> None:
    """Time-sliced logical clients: ``acc (+)= nk * (theta - global)`` in one pass; ``reset`` also returns the replica
    to the global model (theta, bf16 shadow, momentum) for the next co-resident client."""
    load().fold_client(acc, theta, global_w, w_bf16, momentum, float(nk), 1 if first else 0, reset)


def fold_finish(acc: torch.Tensor, theta: torch.Tensor, global_w: torch.Tensor, total: float) -> None:
    """``theta = global + acc / total``: the sample-weighted mean replica this GPU uploads for its logical clients."""
    load().fold_client(acc, theta, global_w, None, None, 1.0 / float(total), 2, False)


def topk_work(n: int, device) -> torch.Tensor:
    """Scratch of the top-k kernels for an ``n``-element arena (int32; reusable by launches on the same stream)."""
    return torch.zeros(int(load().topk_work_words(int(n))), dtype=torch.int32, device=device)


def topk_pack(theta: torch.Tensor, global_w: torch.Tensor, u: torch.Tensor, k: int, work: torch.Tensor, rowptr: int,
              off: int, val: int, *, ef: bool, wire_fp32: bool, cap: int) -> None:
    """One client's top-k upload (``parallel/compress.py``): ``u = (theta - global) [+ u]`` (``ef``: ``u`` holds the
    residual), the ``k`` largest ``|u|`` (ties: lower index) written as a sparse list at the device addresses ``rowptr``
    (uint32 ``[n / 1024 + 1]``), ``off`` (uint16 ``[cap]``) and ``val`` (``[cap]`` fp32 or bf16); with ``ef`` the
    residual ``u`` becomes 0 on the kept entries."""
    load().topk_pack(theta, global_w, u, bool(ef), int(k), work, int(rowptr), int(off), int(val),
                     0 if wire_fp32 else 1, int(cap))


def topk_fold(theta: torch.Tensor, global_w: torch.Tensor, u: torch.Tensor, k: int, work: torch.Tensor,
              acc: torch.Tensor, nk: float, *, ef: bool, first: bool = False, reset: bool = False,
              w_bf16: Optional[torch.Tensor] = None, momentum: Optional[torch.Tensor] = None) -> None:
    """:func:`fold_client` for a top-k client: the selection of :func:`topk_pack`, then ``acc (+)= nk * topk(u)``, the
    residual update and (``reset``) the replica reset."""
    load().topk_fold(theta, global_w, u, bool(ef), int(k), work, acc, float(nk), bool(first), w_bf16, momentum,
                     bool(reset))


def nonzero_pack(theta: torch.Tensor, global_w: torch.Tensor, work: torch.Tensor, rowptr: int, off: int, val: int, *,
                 wire_fp32: bool, cap: int) -> None:
    """The sparse list of the entries where ``theta != global``, value ``cast(theta - global)`` (at most ``cap``)."""
    load().nonzero_pack(theta, global_w, work, int(rowptr), int(off), int(val), 0 if wire_fp32 else 1, int(cap))


def secagg_encode(theta: torch.Tensor, global_w: Optional[torch.Tensor], w: float, range_: float, frac_bits: int,
                  keys: Sequence[Sequence[int]], signs: Sequence[int], nonce: Sequence[int], counter0: int,
                  out: torch.Tensor, saturated: torch.Tensor) -> None:
    """The masked upload of a secure-aggregation round (``parallel/secagg.py``): ``out[e] = encode(theta[e] -
    global_w[e]) + sum_p signs[p] * ChaCha20(keys[p], counter0 + e / 16, nonce)[e % 16]  (mod 2^32)`` as int32 bits,
    ``saturated[0] +=`` the clamped or non-finite elements.  ``global_w`` None: ``x = theta``.  ``keys``: eight uint32
    words per peer; ``signs``: +1 / -1 per peer."""
    words = [int(k) & 0xFFFFFFFF for key in keys for k in key]
    load().secagg_encode(theta, global_w, float(w), float(range_), int(frac_bits), words, [int(s) for s in signs],
                         [int(x) & 0xFFFFFFFF for x in nonce], int(counter0), out, saturated)


def dp_clip_factor(theta: torch.Tensor, global_w: torch.Tensor, clip: float, work: torch.Tensor, s_out: torch.Tensor,
                   norm_out: torch.Tensor, *, s_copy_ptr: int = 0, nonfinite: Optional[torch.Tensor] = None) -> None:
    """DP-FedAvg clip factor: ``s_out[0] = min(1, clip / ||theta - global_w||)`` (0 for a non-finite norm, which also
    adds 1 to ``nonfinite``), ``norm_out[0]`` = the norm.  Deterministic (fixed grid and summation order).  ``work``:
    int64 ``[DP_WORK_WORDS]`` of zeros, reusable by launches on the same stream.  ``s_copy_ptr``: device address that
    receives a second copy of ``s`` (the collective's clip page)."""
    load().dp_clip_factor(theta, global_w, float(clip), work, s_out, norm_out, int(s_copy_ptr), nonfinite)


def fold_client_scaled(acc: torch.Tensor, theta: torch.Tensor, global_w: torch.Tensor, s: torch.Tensor, *,
                       first: bool = False, reset: bool = False, w_bf16: Optional[torch.Tensor] = None,
                       momentum: Optional[torch.Tensor] = None) -> None:
    """:func:`fold_client` with the weight read from the device scalar ``s[0]`` (a DP clip factor): ``acc (+)= s *
    (theta - global)``; ``s == 0`` adds nothing, even where theta is not finite."""
    load().fold_client_scaled(acc, theta, global_w, w_bf16, momentum, s, first, reset)


def cast(src: torch.Tensor, dtype: torch.dtype, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty(src.shape, dtype=dtype, device=src.device)
    load().cast(src.contiguous(), out)
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``src[idx]`` for a resident on-GPU shard (reference: ``X[batch_idxs]``, demo.py:41-42)."""
    if out is None:
        out = torch.empty((idx.numel(),) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    load().gather_rows(src, idx, out)
    return out


AUGMENT_MAX_ROW_BYTES = 48 * 1024      # one image row of gather_augment fits the default dynamic shared memory


def gather_augment(src: torch.Tensor, idx: torch.Tensor, words: torch.Tensor, key: int, padding: int, *,
                   crop: bool = True, flip: bool = True, s0: int = 0, out: Optional[torch.Tensor] = None,
                   mix_rows: Optional[torch.Tensor] = None, batch: Optional[int] = None) -> torch.Tensor:
    """``augment(src[idx])`` for a resident NHWC image shard (bf16 / fp16 / fp32): a random crop of the zero-padded
    image (``padding`` pixels each side) and a random horizontal flip, drawn for output position ``s0 + s`` from
    Philox4x32-10 under the 64-bit ``key`` with counter ``(s0 + s, epoch, stream_lo, stream_hi)``.  ``words`` is a
    device int32 tensor ``{epoch, stream_lo, stream_hi}`` read when the kernel runs (a captured graph follows its
    contents).  ``data/augment.py: gather_augment_reference`` is the same function in torch.

    ``mix_rows`` (device int32 ``[n_batches, 8]``, read when the kernel runs) with ``batch``: mixup / CutMix
    (``data/mix.py``).  Every image is then mixed with its partner in its batch of ``batch`` positions, under the mix
    row ``mix_rows[(s0 + s) // batch]``.  The call must cover whole batches (``s0 % batch == 0``); only the last may be
    short.  Each output is ``mix_batch_reference`` of the augmented batch."""
    if src.dim() != 4 or not src.is_contiguous() or src.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError("gather_augment needs a contiguous NHWC bf16 / fp16 / fp32 shard, got {} {}".format(
            tuple(src.shape), src.dtype))
    H, W, C = src.shape[1:]
    if W * C * src.element_size() > AUGMENT_MAX_ROW_BYTES:
        raise ValueError("gather_augment: an image row is {} bytes, at most {} are supported".format(
            W * C * src.element_size(), AUGMENT_MAX_ROW_BYTES))
    if not 0 <= int(padding) < 1 << 15:
        raise ValueError("gather_augment: padding must be in [0, 32768), got {!r}".format(padding))
    if words.dtype != torch.int32 or words.numel() < 3 or words.device != src.device:
        raise ValueError("gather_augment: words must be an int32 device tensor {epoch, stream_lo, stream_hi}")
    if idx.dtype != torch.int64 or idx.device != src.device:
        raise ValueError("gather_augment: idx must be an int64 tensor on the shard's device")
    if out is None:
        out = torch.empty((idx.numel(), H, W, C), dtype=src.dtype, device=src.device)
    key = int(key) & 0xFFFFFFFFFFFFFFFF
    if mix_rows is not None:
        if batch is None or int(batch) < 1 or int(s0) % int(batch):
            raise ValueError("gather_augment: mixing needs the batch size, and s0 = {} on a batch boundary".format(s0))
        if mix_rows.dtype != torch.int32 or mix_rows.device != src.device or not mix_rows.is_contiguous():
            raise ValueError("gather_augment: mix_rows must be a contiguous int32 tensor on the shard's device")
        load().gather_mix(src, idx.contiguous(), out, words, mix_rows, int(batch),
                          key - (1 << 64) if key >> 63 else key, int(padding), bool(crop), bool(flip), int(s0))
        return out
    load().gather_augment(src, idx.contiguous(), out, words, key - (1 << 64) if key >> 63 else key, int(padding),
                          bool(crop), bool(flip), int(s0))
    return out


def colsum_(x2d: torch.Tensor, out: torch.Tensor, accumulate: bool = True) -> torch.Tensor:
    load().colsum(x2d, out, x2d.shape[0], x2d.shape[1], accumulate)
    return out


def add(a: torch.Tensor, b: torch.Tensor, relu: bool = False) -> torch.Tensor:
    out = torch.empty_like(a)
    load().add_bf16(a, b, out, relu)
    return out


def relu_bwd(y: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    dx = torch.empty_like(dy)
    load().relu_bwd(y, dy, dx)
    return dx


def gelu(x: torch.Tensor) -> torch.Tensor:
    y = torch.empty_like(x)
    load().gelu(x, y)
    return y


def gelu_bwd(x: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    dx = torch.empty_like(x)
    load().gelu_bwd(x, dy, dx)
    return dx


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    """Exact GELU ``x Phi(x)`` of a bf16 tensor (``torch.nn.GELU()``)."""
    y = torch.empty_like(x)
    load().gelu_erf(x, y)
    return y


def gelu_erf_bwd(x: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """``dy (Phi(x) + x phi(x))``, the gradient of :func:`gelu_erf` at ``x``."""
    dx = torch.empty_like(x)
    load().gelu_erf_bwd(x, dy, dx)
    return dx


def pad_rows(src2d: torch.Tensor, kp: int, out: Optional[torch.Tensor] = None, gate: Optional[dict] = None) -> torch.Tensor:
    """``gate`` (bcast_gemm): ``{"flags", "epoch_word", "elem_off", "tile_elems"}`` -- wait for the FedAvg collective's
    arrival flags over the source slice of the bf16 arena before reading it."""
    rows, k = src2d.shape
    if out is None:
        out = torch.empty((rows, kp), dtype=BF16, device=src2d.device)
    g = gate or {}
    load().pad_rows(src2d, out, rows, k, kp, g.get("flags"), g.get("epoch_word"), int(g.get("elem_off", 0)),
                    int(g.get("tile_elems", 0)))
    return out


# ---------------------------------------------------------------------------- conv plumbing
def conv_out_size(h: int, k: int, stride: int, pad: int) -> int:
    return (h + 2 * pad - k) // stride + 1


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def im2col_k(kh: int, kw: int, c: int) -> int:
    """K of an explicit im2col GEMM: the ``kh*kw*C`` taps zero-padded to a multiple of 8 (16-byte TMA rows)."""
    return round_up(kh * kw * c, 8)


def im2col(x: torch.Tensor, kh: int, kw: int, stride: int, pad: int) -> Tuple[torch.Tensor, int, int, int]:
    """NHWC ``x`` -> ``col[N*Ho*Wo, Kp]`` with ``Kp = im2col_k(kh, kw, C)``."""
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
    kp = im2col_k(kh, kw, c)
    col = torch.empty((n * ho * wo, kp), dtype=BF16, device=x.device)
    load().im2col(x, col, n, h, w, c, kh, kw, stride, pad, ho, wo, kp)
    return col, ho, wo, kp


class ConvPlan(collections.namedtuple("ConvPlan", "n h w c cout kh kw stride pad form ho wo M K tap dgrad")):
    """:func:`conv_plan` of one convolution: its geometry, the ``form`` of its forward GEMM, the output size, that
    GEMM's ``M`` and ``K``, the ``tap`` index (``"centre"`` only, else ``None``) and the input gradient's ``dgrad``."""
    __slots__ = ()

    def weight(self, w2d: torch.Tensor) -> torch.Tensor:
        """B operand of the forward and dgrad GEMMs: ``w2d [Cout, kh*kw*Cin]`` itself, or its centre-tap slice."""
        return w2d.view(self.cout, self.kh * self.kw, self.c)[:, self.tap, :] if self.form == "centre" else w2d


@functools.lru_cache(maxsize=None)      # pure: every call with one shape shares one plan
def conv_plan(n: int, h: int, w: int, c: int, cout: int, kh: int, kw: int, stride: int, pad: int) -> ConvPlan:
    """GEMM lowering of a convolution of NHWC ``[n, h, w, c]`` into ``cout`` channels, for training, its backward,
    the fused BatchNorm statistics and evaluation alike.  ``form``:
    * ``"centre"``: a k x k convolution (odd k > 1, "same" padding) over a 1x1 map only ever sees its centre tap --
      every other tap multiplies zero padding.  Exact, and it turns the deepest ResNet stage (32x32 inputs: layer4 is
      1x1) into plain ``[N, Cin] x [Cout, Cin]`` GEMMs on a strided weight view: no im2col / col2im, 9x less K.
    * ``"pointwise"``: 1x1, stride 1, pad 0: a plain GEMM on ``x.view(-1, C)``.
    * ``"implicit"`` (``C % 64 == 0``): A gathered from ``x`` inside the GEMM (:func:`conv_igemm_fwd`, which may
      decline at run time: then ``"im2col"`` runs), no col buffer; the wgrad gathers ``im2col(x)`` on the fly.
    * ``"im2col"``: explicit im2col / col2im + GEMM for the rest (the C = 3 stem, ``Cin % 64 != 0``).
    ``dgrad``: ``"implicit"`` (:func:`conv_igemm_dgrad`, which may decline: then ``"col2im"``) for implicit
    convolutions of stride 2 or of stride 1 and square k > 1; else the dgrad GEMM then ``"view"`` or ``"col2im"``."""
    ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
    tap = None
    if h == 1 and w == 1 and kh == kw and kh % 2 == 1 and kh > 1 and pad == kh // 2 and c % 8 == 0:
        form, K, tap = "centre", c, (kh // 2) * kw + kw // 2
    elif kh == 1 and kw == 1 and stride == 1 and pad == 0 and c % 8 == 0:
        form, K = "pointwise", c
    elif c % 64 == 0:
        form, K = "implicit", kh * kw * c
    else:
        form, K = "im2col", im2col_k(kh, kw, c)
    dgrad = "view" if form in ("centre", "pointwise") else "col2im"
    if form == "implicit" and (stride == 2 or (stride == 1 and kh == kw and kh > 1)):
        dgrad = "implicit"
    return ConvPlan(n, h, w, c, cout, kh, kw, stride, pad, form, ho, wo, n * ho * wo, K, tap, dgrad)


def conv_fwd(x: torch.Tensor, w2d: torch.Tensor, plan: ConvPlan, form: Optional[str] = None,
             col_stats: Optional[torch.Tensor] = None, gate: Optional[dict] = None,
             affine: Optional[dict] = None) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
    """``plan``'s forward GEMM (or ``form``'s) on NHWC ``x`` and channels_last ``w2d``: ``(y [M, Cout] or None when it
    declines, the A operand the wgrad reads)``.  ``col_stats`` / ``affine``: as in :func:`gemm`; ``gate`` (bcast_gemm,
    pointwise and im2col forms): the TMA producer acquires the FedAvg arrival flags over ``w2d``."""
    form = form or plan.form
    if form == "implicit":
        return conv_igemm_fwd(x, w2d, plan.kh, plan.kw, plan.stride, plan.pad, col_stats=col_stats, affine=affine), x
    a = im2col(x, plan.kh, plan.kw, plan.stride, plan.pad)[0] if form == "im2col" else x.view(plan.M, plan.c)
    gk = {}
    if gate is not None and form != "centre":
        gk = dict(flags=gate["flags"], flag_epoch_word=gate["epoch_word"], flag_elem_off=gate["elem_off"],
                  flag_tile_elems=gate["tile_elems"], force_bn=pick_bn(a.shape[0], w2d.shape[0]))
    return gemm(a, plan.weight(w2d), col_stats=col_stats, affine=affine, **gk), a


HALO_BM = 64                      # output pixels of one halo-kernel tile (conv_halo.cu)
_HALO_MAX_SMEM = 227 * 1024       # shared memory one H100 block may use
_HALO_FORMS = ((1, 64), (1, 128), (2, 64))   # (stride, gathered channels) conv_halo.cu instantiates; stride 2: forward


def halo_smem_bytes(h: int, w: int, c: int = 64, stride: int = 1) -> int:
    """Shared memory of the halo kernel over an ``h x w`` input of ``c`` gathered channels at ``stride``: ``c / 64``
    halo boxes of the ``64 / (ho wo)`` images (each rounded up to 1 KB), ``9 c / 64`` 8 KB weight slots, one mbarrier
    per slot plus one for the halo (padded to a multiple of 16), column statistics and the 1 KB realignment
    (conv_halo.cu halo_fixed_bytes)."""
    ho, wo = conv_out_size(h, 3, stride, 1), conv_out_size(w, 3, stride, 1)
    box = (HALO_BM // (ho * wo)) * (stride * (ho - 1) + 3) * (stride * (wo - 1) + 3) * 128
    k_tiles = 9 * (c // 64)
    return c // 64 * round_up(box, 1024) + k_tiles * 8192 + round_up(1 + k_tiles, 16) * 8 + 4 * 64 * 4 + 1024


def halo_eligible(kh: int, kw: int, stride: int, pad: int, c: int, h: int, w: int,
                  affine: Optional[dict] = None, dgrad: bool = False) -> bool:
    """Whether the halo-tiled kernel takes a convolution over an ``h x w`` input: 3x3, pad 1, a (stride, gathered
    channels) form of ``_HALO_FORMS`` -- stride 1 over 64 or 128 channels of the gathered tensor (``x`` forward, ``dy``
    dgrad), or stride 2 over a 64-channel ``x`` (forward only) --, a 64-row tile holds whole output images, the halo
    and the ``9 c / 64`` weight slots fit in shared memory, and no eval-mode ``affine`` epilogue is asked for."""
    if kh != 3 or kw != 3 or pad != 1 or (stride, c) not in _HALO_FORMS or (dgrad and stride != 1):
        return False
    hw = conv_out_size(h, 3, stride, 1) * conv_out_size(w, 3, stride, 1)
    return (hw <= HALO_BM and HALO_BM % hw == 0 and affine is None and
            halo_smem_bytes(h, w, c, stride) <= _HALO_MAX_SMEM)


def halo_cluster(m_rows: int) -> int:
    """CTAs of a halo-kernel cluster along M sharing the weight tiles: 4, or 2 / 1 when the tile count does not divide.
    At the layer2 shapes (batch 128), clusters of 1, 2, 4 and 8 were within 0.25 us of each other; 4 was fastest or
    tied for the stride-1 GEMMs (scripts/conv_halo_wide_bench.py, one H100 80GB HBM3 at 700 W)."""
    tiles = (m_rows + HALO_BM - 1) // HALO_BM
    return 4 if tiles % 4 == 0 else 2 if tiles % 2 == 0 else 1


_SMALLMAP_FORMS = ((1, 256), (2, 128))   # (stride, gathered channels) of conv_smallmap; stride 2: forward only
SMALLMAP_BN = 32                          # output columns of one image-tile CTA: all 36 weight k-tiles fit


def smallmap_smem_bytes(h: int, w: int, c: int = 256, stride: int = 1, bn: int = SMALLMAP_BN) -> int:
    """Shared memory of the image-tile kernel over an ``h x w`` input of ``c`` gathered channels at ``stride``:
    ``c / 64`` boxes of the ``64 / (ho wo)`` whole input images (no halo; each rounded up to 1 KB), ``9 c / 64``
    weight slots of ``bn x 64`` bf16, one mbarrier per slot plus one for the images (padded to a multiple of 16),
    column statistics, the 128-byte zero line of the out-of-image taps and the 1 KB realignment (conv_halo.cu
    halo_fixed_bytes)."""
    ho, wo = conv_out_size(h, 3, stride, 1), conv_out_size(w, 3, stride, 1)
    box = (HALO_BM // (ho * wo)) * h * w * 128
    k_tiles = 9 * (c // 64)
    return (c // 64 * round_up(box, 1024) + k_tiles * bn * 128 + round_up(1 + k_tiles, 16) * 8 + 4 * bn * 4 + 128
            + 1024)


def smallmap_eligible(kh: int, kw: int, stride: int, pad: int, c: int, h: int, w: int,
                      affine: Optional[dict] = None, dgrad: bool = False) -> bool:
    """Whether the image-tile kernel (``conv_smallmap``) takes a convolution over an ``h x w`` input: 3x3, pad 1, a
    (stride, gathered channels) form of ``_SMALLMAP_FORMS`` -- stride 1 over 256 channels of the gathered tensor
    (``x`` forward, ``dy`` dgrad) or stride 2 over a 128-channel ``x`` (forward only) --, a 64-row tile holds whole
    output images, the images and the weight slots fit in shared memory, and no eval-mode ``affine`` epilogue."""
    if kh != 3 or kw != 3 or pad != 1 or (stride, c) not in _SMALLMAP_FORMS or (dgrad and stride != 1):
        return False
    hw = conv_out_size(h, 3, stride, 1) * conv_out_size(w, 3, stride, 1)
    return (hw <= HALO_BM and HALO_BM % hw == 0 and affine is None and
            smallmap_smem_bytes(h, w, c, stride) <= _HALO_MAX_SMEM)


def _conv_path(path: Optional[str], eligible: bool, smallmap: bool = False) -> str:
    if path is None:
        return "halo" if eligible else "smallmap" if smallmap else "im2col"
    if path not in ("halo", "smallmap", "im2col"):
        raise ValueError("path must be None, 'halo', 'smallmap' or 'im2col', not {!r}".format(path))
    if path == "halo" and not eligible:
        raise ValueError("the halo kernel does not take this convolution (see halo_eligible)")
    if path == "smallmap" and not smallmap:
        raise ValueError("the image-tile kernel does not take this convolution (see smallmap_eligible)")
    return path


def conv_igemm_fwd(x: torch.Tensor, w2d: torch.Tensor, kh: int, kw: int, stride: int, pad: int,
                   col_stats: Optional[torch.Tensor] = None, affine: Optional[dict] = None,
                   cluster_k: Optional[int] = None, force_bn: int = 0,
                   out: Optional[torch.Tensor] = None, path: Optional[str] = None,
                   mc: Optional[int] = None, bn: int = SMALLMAP_BN) -> Optional[torch.Tensor]:
    """Implicit-GEMM convolution forward: ``y[N*Ho*Wo, Cout]`` straight from NHWC ``x`` through TMA
    im2col loads (no ``col`` buffer).  ``w2d``: ``[Cout, kh*kw*Cin]`` channels_last weights.  ``affine``: eval-mode
    BatchNorm epilogue as in :func:`gemm`.  ``out``: contiguous bf16 ``[N*Ho*Wo, Cout]`` to write.  Returns ``None``
    when the shape (or the epilogue) is not supported (Cin % 64 != 0).

    ``path``: ``None`` takes the halo-tiled kernel whenever :func:`halo_eligible` holds, else the image-tile kernel
    whenever :func:`smallmap_eligible` holds, else the im2col-mode kernel; ``"halo"`` / ``"smallmap"`` /
    ``"im2col"`` force one (``"halo"`` or ``"smallmap"`` on a shape that kernel does not take raises).
    ``mc``: cluster size of the halo and image-tile kernels (default :func:`halo_cluster`); ``bn``: output columns
    per image-tile CTA (32, or 64 at the stride-2 form); ``cluster_k`` / ``force_bn`` apply to the im2col path."""
    n, h, w, c = x.shape
    cout = w2d.shape[0]
    if c % 64 or w2d.shape[1] != kh * kw * c or not x.is_contiguous() or not w2d.is_contiguous():
        return None
    ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
    M, K = n * ho * wo, kh * kw * c
    halo = halo_eligible(kh, kw, stride, pad, c, h, w, affine) and cout % 8 == 0
    small = smallmap_eligible(kh, kw, stride, pad, c, h, w, affine) and cout % bn == 0
    kind = _conv_path(path, halo, small)
    if kind == "halo":
        y = out if out is not None else torch.empty((M, cout), dtype=BF16, device=x.device)
        if not load().conv_halo(x, w2d, y, stride, False, mc or halo_cluster(M), col_stats):
            raise RuntimeError("conv_halo declined a convolution halo_eligible admits")
        return y
    if kind == "smallmap":
        y = out if out is not None else torch.empty((M, cout), dtype=BF16, device=x.device)
        if not load().conv_smallmap(x, w2d, y, stride, False, mc or halo_cluster(M), bn, col_stats):
            raise RuntimeError("conv_smallmap declined a convolution smallmap_eligible admits")
        return y
    bn = force_bn or pick_bn(M, cout)
    if cluster_k is None:
        cluster_k = pick_cluster_k(M, cout, K, bn)
    y = out if out is not None else torch.empty((M, cout), dtype=BF16, device=x.device)
    af = affine or {}
    ok = load().conv_igemm_fwd(x, w2d, y, kh, kw, stride, pad, ho, wo, cluster_k, bn, col_stats, af.get("scale"),
                               af.get("shift"), af.get("residual"), bool(af.get("relu", False)))
    return y if ok else None


S2_MAX_TAPS = 4     # taps of one parity class the stride-2 dgrad kernel takes (gemm_wgmma.cu S2_MAX_TAPS)


def conv_s2_dgrad_taps(kh: int, kw: int, pad: int, ho: int, wo: int) -> Optional[List[List[Tuple[int, int, int]]]]:
    """Sub-pixel decomposition of the input gradient of a stride-2 convolution with dy of size ``ho x wo``.

    Class ``c = 2a + b`` holds the dx pixels ``(2i + a, 2j + b)``; its entry lists the taps ``(r * kw + s, dp, dq)``
    with ``dx[2i + a, 2j + b] = sum dy[i + dp, j + dq] * W[r, s]`` (``2 (i + dp) - pad + r = 2i + a``), terms with
    ``dy`` outside the image being zero.  Taps whose dy pixel lies past dy for every ``i`` / ``j`` are left out.
    ``None`` when a class needs a negative offset or more than ``S2_MAX_TAPS`` taps."""
    classes = []
    for a in (0, 1):
        for b in (0, 1):
            taps = []
            for r in range(kh):
                if (a + pad - r) % 2:
                    continue
                dp = (a + pad - r) // 2
                for s in range(kw):
                    if (b + pad - s) % 2:
                        continue
                    dq = (b + pad - s) // 2
                    if dp < 0 or dq < 0:
                        return None
                    if dp < ho and dq < wo:
                        taps.append((r * kw + s, dp, dq))
            if len(taps) > S2_MAX_TAPS:
                return None
            classes.append(taps)
    return classes


def conv_igemm_dgrad(dy: torch.Tensor, w2d: torch.Tensor, in_shape, kh: int, kw: int, pad: int, stride: int = 1,
                     out: Optional[torch.Tensor] = None, path: Optional[str] = None,
                     mc: Optional[int] = None, cluster_k: Optional[int] = None) -> Optional[torch.Tensor]:
    """Implicit-GEMM input gradient of a stride-1 or stride-2 convolution: ``dx[N, H, W, Cin]`` from NHWC ``dy`` and
    the channels_last weights ``w2d [Cout, kh*kw*Cin]``, gathered by TMA im2col, with the weight slab of each tap
    loaded MN-major in place (no ``dcol`` buffer, no col2im, no weight transpose).  Stride 1: the flipped-filter
    convolution of ``dy``.  Stride 2: one launch over the four parity classes of :func:`conv_s2_dgrad_taps`.
    ``out``: contiguous bf16 ``[N, H, W, Cin]`` to write (every element is written).  Returns ``None`` when the shape
    is not supported (channels not multiples of 64, other strides).  ``path`` / ``mc``: as in :func:`conv_igemm_fwd`
    (the halo and image-tile kernels gather ``dy``, so ``Cout`` is what their rules check).  ``cluster_k``: cluster
    split-K of the stride-1 im2col path (default :func:`pick_cluster_k`)."""
    n, h, w, c = in_shape
    cout = dy.shape[-1]
    if c % 64 or cout % 64 or w2d.shape[1] != kh * kw * c or not dy.is_contiguous() or not w2d.is_contiguous():
        return None
    kind = _conv_path(path, halo_eligible(kh, kw, stride, pad, cout, h, w, dgrad=True),
                      smallmap_eligible(kh, kw, stride, pad, cout, h, w, dgrad=True) and c % SMALLMAP_BN == 0)
    if kind == "halo":
        dx = out if out is not None else torch.empty((n, h, w, c), dtype=BF16, device=dy.device)
        if not load().conv_halo(dy, w2d, dx, 1, True, mc or halo_cluster(n * h * w), None):
            raise RuntimeError("conv_halo declined a convolution halo_eligible admits")
        return dx
    if kind == "smallmap":
        dx = out if out is not None else torch.empty((n, h, w, c), dtype=BF16, device=dy.device)
        if not load().conv_smallmap(dy, w2d, dx, 1, True, mc or halo_cluster(n * h * w), SMALLMAP_BN, None):
            raise RuntimeError("conv_smallmap declined a convolution smallmap_eligible admits")
        return dx
    if stride == 1:
        M, K = n * h * w, kh * kw * cout
        bn = pick_bn(M, c)
        dx = out if out is not None else torch.empty((n, h, w, c), dtype=BF16, device=dy.device)
        if cluster_k is None:
            cluster_k = pick_cluster_k(M, c, K, bn)
        ok = load().conv_igemm_dgrad(dy, w2d, dx, kh, kw, pad, cluster_k, bn)
        return dx if ok else None
    if stride != 2:
        return None
    ho, wo = dy.shape[1], dy.shape[2]
    classes = conv_s2_dgrad_taps(kh, kw, pad, ho, wo)
    if classes is None:
        return None
    bn = pick_bn(4 * n * ho * wo, c)       # rows of all four classes
    words = [[t | dp << 16 | dq << 24 for t, dp, dq in taps] + [0] * (S2_MAX_TAPS - len(taps)) for taps in classes]
    dx = out if out is not None else torch.empty((n, h, w, c), dtype=BF16, device=dy.device)
    ok = load().conv_igemm_dgrad_s2(dy, w2d, dx, kh, kw, [len(t) for t in classes], [x for ws in words for x in ws], bn)
    return dx if ok else None


def conv_igemm_wgrad_(dy2d: torch.Tensor, x: torch.Tensor, dw2d: torch.Tensor, kh: int, kw: int, stride: int,
                      pad: int, sgd: Optional[dict] = None) -> bool:
    """Implicit wgrad: ``dw2d[Cout, kh*kw*Cin] += dy2d^T im2col(x)`` (fp32 atomics, split over
    pixels) without materialising ``im2col(x)``.  ``sgd``: optimizer epilogue as in :func:`gemm`.  False: nothing
    was done (shape not supported, or the optimizer epilogue declined)."""
    n, h, w, c = x.shape
    cout = dy2d.shape[1]
    if c % 64 or not x.is_contiguous() or not dy2d.is_contiguous() or not dw2d.is_contiguous():
        return False
    ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
    M, K = n * ho * wo, kh * kw * c
    bn = pick_bn(cout, K)
    split_k = pick_split_k(cout, K, M, bn)
    if sgd is not None and split_k != 1:
        return False                # the optimizer epilogue needs every tile's complete gradient in one CTA
    sg = sgd or {}
    return bool(load().conv_igemm_wgrad(dy2d, x, dw2d, cout, kh, kw, stride, pad, ho, wo, split_k, bn,
                                        sg.get("theta"), sg.get("theta_bf16"), sg.get("momentum"), sg.get("hyper"),
                                        bool(sg.get("nesterov", False)), sg.get("anchor"), sg.get("corr"),
                                        sg.get("adam_v")))


def col2im(col: torch.Tensor, shape: Tuple[int, int, int, int], kh: int, kw: int, stride: int, pad: int,
           ho: int, wo: int) -> torch.Tensor:
    n, h, w, c = shape
    dx = torch.empty(shape, dtype=BF16, device=col.device)
    load().col2im(col, dx, n, h, w, c, kh, kw, stride, pad, ho, wo, col.shape[1])
    return dx


def maxpool(x: torch.Tensor, k: int, stride: int, pad: int) -> Tuple[torch.Tensor, torch.Tensor]:
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, k, stride, pad), conv_out_size(w, k, stride, pad)
    y = torch.empty((n, ho, wo, c), dtype=BF16, device=x.device)
    # winners: one byte (tap index inside the window) on the 16-byte path, a flat int32 position otherwise
    arg = torch.empty((n, ho, wo, c), dtype=torch.uint8 if (c % 8 == 0 and k * k <= 255) else torch.int32, device=x.device)
    load().maxpool(x, y, arg, n, h, w, c, k, stride, pad, ho, wo)
    return y, arg


def maxpool_bwd(dy: torch.Tensor, arg: torch.Tensor, in_shape, k: int, stride: int, pad: int,
                dy_b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``dy_b``: optional second piece of the gradient (summed while loading; byte-argmax path only)."""
    n, h, w, c = in_shape
    if dy_b is not None and arg.dtype != torch.uint8:
        dy, dy_b = add(dy, dy_b), None
    dx = torch.empty(in_shape, dtype=BF16, device=dy.device)
    load().maxpool_bwd(dy, dy_b, arg, dx, n, h, w, c, dy.shape[1], dy.shape[2], k, stride, pad)
    return dx


def bn_relu_maxpool(z: torch.Tensor, sums: torch.Tensor, gamma, beta, rmean, rvar, nbt, eps: float, momentum: float,
                    k: int, stride: int, pad: int):
    """ResNet stem in one pass: ``maxpool(relu(batchnorm(z)))`` from the conv output ``z`` (NHWC bf16) and the batch
    statistic sums the conv GEMM's epilogue accumulated, without materialising the normalised activation.
    -> ``(p, argmax_u8, save_mean, save_rstd)`` or ``None`` when the shape is not supported (callers fall back to
    ``bn_apply`` + ``maxpool``).  Training mode only."""
    n, h, w, c = z.shape
    if c % 8 or k * k > 255:
        return None
    ho, wo = conv_out_size(h, k, stride, pad), conv_out_size(w, k, stride, pad)
    p = torch.empty((n, ho, wo, c), dtype=BF16, device=z.device)
    arg = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=z.device)
    mean = torch.empty(c, dtype=torch.float32, device=z.device)
    rstd = torch.empty(c, dtype=torch.float32, device=z.device)
    if not load().bn_relu_maxpool(z, p, arg, sums, gamma, beta, rmean, rvar, mean, rstd, nbt, n, h, w, c, k, stride, pad,
                                  ho, wo, eps, momentum):
        return None
    return p, arg, mean, rstd


def bn_maxpool_bwd(z: torch.Tensor, p: torch.Tensor, arg: torch.Tensor, dy_a: torch.Tensor, dy_b: Optional[torch.Tensor],
                   gamma, mean: torch.Tensor, rstd: torch.Tensor, sums_b: torch.Tensor, dgamma, dbeta, k: int, stride: int,
                   pad: int) -> Optional[torch.Tensor]:
    """Backward of :func:`bn_relu_maxpool`: ``dz`` from the pooled gradient ``dy_a (+ dy_b)``; ``dgamma`` / ``dbeta``
    are accumulated in place.  ``sums_b``: zeroed ``[2 * C]`` fp32 scratch.  ``None`` = shape not supported."""
    n, h, w, c = z.shape
    dz = torch.empty_like(z)
    if not load().bn_maxpool_bwd(z, p, arg, dy_a, dy_b, dz, gamma, mean, rstd, sums_b, dgamma, dbeta, n, h, w, c, k, stride,
                                 pad, p.shape[1], p.shape[2]):
        return None
    return dz


def gn_work(n: int, c: int, groups: int, device) -> torch.Tensor:
    """Scratch of :func:`gn_bwd`: fp32 ``[G + 2 N C]``, per-group arrival counters then per-sample channel partials.  The
    counters must be zero when the backward starts: :func:`gn_fwd` zeroes them when it is given the buffer, and the
    backward leaves them zero, so one buffer serves any number of launches on one stream."""
    return torch.empty(groups + 2 * n * c, dtype=torch.float32, device=device)


def gn_fwd(z: torch.Tensor, residual: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor, groups: int,
           eps: float = 1e-5, relu: bool = False, work: Optional[torch.Tensor] = None):
    """GroupNorm of NHWC bf16 ``z`` with ``groups`` contiguous channel blocks, plus the residual and the ReLU:
    ``y = relu(gamma_c * (z - mean_ng) * rstd_ng + beta_c + residual)``, biased variance, statistics in fp32.
    -> ``(y, mean, rstd)`` with fp32 ``[N, G]`` statistics.  ``work``: the backward's :func:`gn_work` buffer, if any."""
    n = z.shape[0]
    y = torch.empty_like(z)
    mean = torch.empty((n, groups), dtype=torch.float32, device=z.device)
    rstd = torch.empty((n, groups), dtype=torch.float32, device=z.device)
    load().gn_fwd(z, None if residual is None else residual.contiguous(), y, gamma, beta, mean, rstd, int(groups),
                  float(eps), bool(relu), work)
    return y, mean, rstd


def gn_bwd(z: torch.Tensor, y: torch.Tensor, dy_a: torch.Tensor, dy_b: Optional[torch.Tensor], gamma: torch.Tensor,
           mean: torch.Tensor, rstd: torch.Tensor, dgamma: Optional[torch.Tensor], dbeta: Optional[torch.Tensor],
           groups: int, relu: bool = False, want_dres: bool = False, work: Optional[torch.Tensor] = None):
    """Backward of :func:`gn_fwd` from the gradient ``dy_a (+ dy_b)`` of ``y``: -> ``(dz, dres)`` where ``dres`` (the
    residual's gradient, ``dy'`` after the ReLU mask) is ``None`` unless ``want_dres``.  ``dgamma`` / ``dbeta`` (fp32
    ``[C]``) are ACCUMULATED, in a fixed summation order.  ``work``: a :func:`gn_work` buffer with zero counters (a
    fresh zeroed one when ``None``)."""
    n, c = z.shape[0], z.shape[3]
    if work is None:
        work = torch.zeros(groups + 2 * n * c, dtype=torch.float32, device=z.device)
    dz = torch.empty_like(z)
    dres = torch.empty_like(z) if want_dres else None
    load().gn_bwd(z, y, dy_a.contiguous(), None if dy_b is None else dy_b.contiguous(), dz, dres, gamma, mean, rstd,
                  dgamma, dbeta, int(groups), bool(relu), work)
    return dz, dres


def avgpool(x: torch.Tensor) -> torch.Tensor:
    n, h, w, c = x.shape
    y = torch.empty((n, c), dtype=BF16, device=x.device)
    load().avgpool(x, y, n, h * w, c)
    return y


def avgpool_bwd(dy: torch.Tensor, in_shape) -> torch.Tensor:
    n, h, w, c = in_shape
    dx = torch.empty(in_shape, dtype=BF16, device=dy.device)
    load().avgpool_bwd(dy, dx, n, h * w, c)
    return dx


# ---------------------------------------------------------------------------- losses
def softmax_xent(logits: torch.Tensor, target: torch.Tensor, want_grad: bool = True,
                 grad_dtype: Optional[torch.dtype] = None, acc: Optional[torch.Tensor] = None,
                 loss_scale: Optional[float] = None, mix_row: Optional[torch.Tensor] = None, smoothing: float = 0.0):
    """Fused softmax cross-entropy: returns ``(acc, dlogits)`` where ``acc[0]`` is the
    batch-mean loss and ``acc[1]`` the number of correct predictions.  ``acc`` (fp32 ``[2]``) may be supplied: the
    kernel ADDS into it (a device-side running sum over the steps of an epoch, no extra kernels).  ``loss_scale``
    replaces the ``1 / rows`` that scales the loss and the gradient (1.0: the sum of the row losses).

    ``mix_row`` (the step's device int32 mix row) and ``smoothing``: the soft target of ``data/mix.py``, the partner
    of row ``r`` being row ``r - 1`` (mod rows) of ``target``; ``acc[1]`` then adds the lam-weighted hits."""
    rows, c = logits.shape
    if acc is None:
        acc = torch.zeros(2, dtype=torch.float32, device=logits.device)
    dl = torch.empty_like(logits, dtype=grad_dtype or logits.dtype) if want_grad else None
    scale = 1.0 / rows if loss_scale is None else loss_scale
    if mix_row is None and smoothing == 0.0:
        load().softmax_xent(logits, target, dl, acc, rows, c, logits.stride(0), scale)
    else:
        load().softmax_xent_soft(logits, target, dl, acc, rows, c, logits.stride(0), scale, mix_row, float(smoothing))
    return acc, dl


def linear_xent_head(x: torch.Tensor, w_bf16: torch.Tensor, bias: Optional[torch.Tensor], target: torch.Tensor,
                     dw: torch.Tensor, db: Optional[torch.Tensor], acc: Optional[torch.Tensor] = None,
                     want_dx: bool = True, want_logits: bool = False, mix_row: Optional[torch.Tensor] = None,
                     smoothing: float = 0.0):
    """Classifier head in one launch: ``logits = x w^T + b`` (<= 32 classes), softmax cross-entropy, and the head's whole
    backward -- ``dx`` (bf16), ``dw += dlogits^T x``, ``db += colsum(dlogits)`` (fp32, accumulated in place), the batch-mean
    loss / #correct added into ``acc``.  Returns ``(acc, dx, logits)`` or ``None`` when the shape is not supported.
    ``mix_row`` / ``smoothing``: the soft target, as in :func:`softmax_xent` (no logits output)."""
    rows, K = x.shape
    if acc is None:
        acc = torch.zeros(2, dtype=torch.float32, device=x.device)
    dx = torch.empty((rows, K), dtype=BF16, device=x.device) if want_dx else None
    if mix_row is not None or smoothing != 0.0:
        if want_logits:
            raise ValueError("linear_xent_head: the soft-target head has no logits output")
        ok = load().linear_xent_head_soft(x, w_bf16, bias, target, dx, dw, db, acc, 1.0 / rows, mix_row,
                                          float(smoothing))
        return (acc, dx, None) if ok else None
    logits = torch.empty((rows, w_bf16.shape[0]), dtype=torch.float32, device=x.device) if want_logits else None
    ok = load().linear_xent_head(x, w_bf16, bias, target, dx, dw, db, acc, logits, 1.0 / rows)
    return (acc, dx, logits) if ok else None


def linear_xent_eval(x: torch.Tensor, w_bf16: torch.Tensor, bias: Optional[torch.Tensor], target: torch.Tensor,
                     acc: torch.Tensor, want_logits: bool = False):
    """Forward-only classifier head (evaluation), one launch: ``logits = x w^T + b`` (<= 32 classes), then ``acc[0]``
    += the SUM of the row cross-entropies and ``acc[1]`` += #correct.  Returns ``(acc, logits or None)`` or ``None``
    when the shape is not supported."""
    logits = torch.empty((x.shape[0], w_bf16.shape[0]), dtype=torch.float32, device=x.device) if want_logits else None
    ok = load().linear_xent_eval(x, w_bf16, bias, target, acc, logits)
    return (acc, logits) if ok else None


def mse(pred: torch.Tensor, target: torch.Tensor, want_grad: bool = True):
    acc = torch.zeros(2, dtype=torch.float32, device=pred.device)
    dp = torch.empty_like(pred) if want_grad else None
    load().mse(pred.contiguous(), target.contiguous().float(), dp, acc, 1.0 / pred.numel())
    return acc, dp


# ---------------------------------------------------------------------------- batched GEMM / attention / embedding
def gemm_batched(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int, lda: int, ldb: int,
                 ldd: int, a_mn: bool, b_mn: bool, n_outer: int, n_inner: int, a_strides, b_strides, d_strides,
                 alpha: float = 1.0, act: int = 0, accumulate: bool = False) -> torch.Tensor:
    """Strided-batched wgmma GEMM over a two-level batch (outer, inner) = (batch, head): operands are
    addressed through 4-D TMA tensor maps, so Q/K/V slices of a packed QKV buffer need no copies.
    ``*_strides`` = (outer, inner) element strides; ``a``/``b``/``out`` give the base pointers."""
    load().gemm_batched(a, b, out, M, N, K, lda, ldb, ldd, a_mn, b_mn, act, alpha, n_outer, n_inner,
                        a_strides[0], a_strides[1], b_strides[0], b_strides[1], d_strides[0], d_strides[1], accumulate)
    return out


def embedding_bwd_(dy2d: torch.Tensor, idx: torch.Tensor, grad_table: torch.Tensor) -> None:
    load().embedding_bwd(dy2d, idx, grad_table)


# ---------------------------------------------------------------------------- MXFP8 (block-scaled fp8)
def _sf_bytes(rows: int, k: int) -> int:
    return ((rows + 127) // 128) * ((k + 127) // 128) * 512


def quant_mx_rows(x2d: torch.Tensor):
    """bf16 ``[R, C]`` -> (e4m3 ``[R, Cp]`` as uint8, UE8M0 scale atoms); scales along C."""
    R, C = x2d.shape
    Cp = round_up(C, 16)
    q = torch.empty((R, Cp), dtype=torch.uint8, device=x2d.device)
    sf = torch.empty(_sf_bytes(R, C), dtype=torch.uint8, device=x2d.device)
    load().quant_mx_rows(x2d, q, sf, R, C, x2d.stride(0), Cp)
    return q, sf


def quant_mx_cols(x2d: torch.Tensor):
    """bf16 ``[R, C]`` -> (e4m3 ``[C, Rp]`` = quantised TRANSPOSE, scale atoms); scales along R."""
    R, C = x2d.shape
    Rp = round_up(R, 16)
    q = torch.zeros((C, Rp), dtype=torch.uint8, device=x2d.device) if Rp != R else \
        torch.empty((C, Rp), dtype=torch.uint8, device=x2d.device)
    sf = torch.empty(_sf_bytes(C, R), dtype=torch.uint8, device=x2d.device)
    load().quant_mx_cols(x2d, q, sf, R, C, x2d.stride(0), Rp)
    return q, sf


def gemm_fp8(qa: torch.Tensor, sfa, qb: torch.Tensor, sfb, K: int, *, out: Optional[torch.Tensor] = None,
             out_dtype: torch.dtype = BF16, bias: Optional[torch.Tensor] = None, act: int = 0,
             accumulate: bool = False, alpha: float = 1.0, split_k: int = 1, n_valid: Optional[int] = None):
    """``out[M,N] = act(alpha * (A*SFA) @ (B*SFB)^T + bias)`` with e4m3 operands ``qa [M,Kp]``, ``qb [N,Kp]``.
    ``accumulate`` adds onto ``out``.  With ``split_k > 1`` the K slices add their partial products into ``out`` with
    atomics, so without ``accumulate`` the output is zeroed first."""
    M, N = qa.shape[0], qb.shape[0]
    if n_valid is not None:
        N = min(N, n_valid)
    if out is None:
        out = torch.zeros((M, N), dtype=out_dtype, device=qa.device) if (accumulate or split_k > 1) else \
            torch.empty((M, N), dtype=out_dtype, device=qa.device)
    elif split_k > 1 and not accumulate:
        out.zero_()
    ldd = out.stride(0) if out.dim() == 2 else N
    load().gemm_fp8(qa, qb, out, bias, sfa, sfb, M, N, K, qa.stride(0), qb.stride(0), ldd, act, split_k, accumulate, alpha)
    return out
