"""Host-side plumbing shared by the autograd wrappers: argument checks in the
style of the reference's C++ wrappers (rasterization.cpp:70-85,
dibr_soft_mask.cpp:63-82), workspace allocation, and the library calls."""
import torch

from ... import _lib
# Pointer and stream arguments for calling an entry point by hand; the tests that assert raw status
# codes take them from here.
from ..._lib import ptr, stream_ptr  # noqa: F401


def aligned(t):
    """``t``, or a fresh copy of it if its data does not start on a 16-byte boundary.  The fused
    entry points reject such pointers (their kernels make 16-byte vector accesses); a contiguous
    view at an element offset, e.g. ``buf[1:].view(B, F, 3, 2)``, is still legal input."""
    return t if t is None or t.data_ptr() % 16 == 0 else t.clone()


FEATURE_DTYPES = (torch.float32, torch.bfloat16)   # storage of face_features / interpolated features


def check_feature_dtype(func, name, t):
    if t is not None and t.dtype not in FEATURE_DTYPES:
        raise RuntimeError(f"\"{func}\" not implemented for '{str(t.dtype).replace('torch.', '')}' "
                           f"({name}: kaolin_b200 stores features as float32 or bfloat16)")


def check_tensors(func, named, dtype=torch.float32):
    """All tensors on the same CUDA device with the expected dtype (no CPU path)."""
    dev = None
    for name, t in named:
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{func}: {name} must be a torch.Tensor")
        if not t.is_cuda:
            raise RuntimeError(f"{func}: expected {name} to be a CUDA tensor "
                               "(kaolin_b200 has no CPU path)")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"{func}: expected all tensors on {dev}, {name} is on {t.device}")
        if dtype is not None and t.is_floating_point() and t.dtype != dtype:
            raise RuntimeError(f"\"{func}\" not implemented for '{str(t.dtype).replace('torch.', '')}' "
                               "(kaolin_b200 supports float32 and float64)")
    return dev


def check_float32(func, named):
    """Every tensor is float32.  ``check_tensors`` lets integer and bool tensors through (index
    arguments share its lists); the kernels read these arguments as ``float``, so a tensor of any
    other element type must not reach them."""
    for name, t in named:
        if t is not None and t.dtype != torch.float32:
            raise RuntimeError(f"\"{func}\" not implemented for '{str(t.dtype).replace('torch.', '')}' "
                               f"({name}: kaolin_b200 reads it as float32)")


def check_size(func, name, t, shape):
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"{func}: expected {name} of size {list(shape)}, got {list(t.shape)}")


def any_double(*tensors):
    """Whether a float64 tensor is among the inputs: such calls run the float64 instantiation."""
    return any(isinstance(t, torch.Tensor) and t.dtype == torch.float64 for t in tensors)


def join_features(face_features):
    """-> (face_features as one tensor, split).  A list/tuple of (..., D_i) feature tensors is
    concatenated along the last dimension, and ``split(out)`` cuts an output interpolated from it
    back into a tuple of (..., D_i) views; a single tensor passes through both unchanged."""
    if not isinstance(face_features, (list, tuple)):
        return face_features, lambda out: out

    def split(out):
        outs, cur = [], 0
        for f in face_features:
            outs.append(out[..., cur:cur + f.shape[-1]])
            cur += f.shape[-1]
        return tuple(outs)
    return torch.cat(face_features, dim=-1), split


# Screen tiles that get a soft-mask hit-cache block (forward scratch of the enumerate / evaluate
# kernels AND the backward's input).  Every tile when that fits in CACHE_MAX_BYTES - at 256^2 a third
# of the 16x16 tiles touch the silhouette, at 1024^2 a tenth, and the host cannot know the number
# without a device sync - else as many as fit; tiles beyond the cache take the single-kernel path
# and are recomputed in backward: same results, several times slower.  Both knobs are module
# attributes (a caller with many live forward graphs can lower CACHE_MAX_BYTES); callers that need
# no gradient do not keep the workspace alive (render/mesh/dibr.py).
CACHE_TILE_FRACTION = 1.0
CACHE_MIN_TILES = 64
CACHE_MAX_BYTES = 4 << 30


def cache_tiles_for(batch, height, width, knum):
    """How many 16x16 tiles get a soft-mask hit-cache block (3072*knum + 16 bytes each)."""
    tiles = batch * ((height + 15) // 16) * ((width + 15) // 16)
    want = max(CACHE_MIN_TILES, int(tiles * CACHE_TILE_FRACTION))
    return min(tiles, want, max(1, CACHE_MAX_BYTES // (3072 * knum + 16)))


_ws_bytes = {}     # (batch, faces, H, W, knum, cache policy, f64) -> bytes: a pure function of the shape


def workspace(batch, total_faces, height, width, device, knum=0, f64=False):
    key = (batch, total_faces, height, width, knum, CACHE_TILE_FRACTION, CACHE_MAX_BYTES, f64)
    n = _ws_bytes.get(key)
    if n is None:
        if f64:         # the float64 kernels keep no hit cache
            n = _lib.lib().dibr_b200_workspace_bytes_f64(batch, total_faces, height, width)
        elif knum > 0:
            want = cache_tiles_for(batch, height, width, knum)
            n = _lib.lib().dibr_b200_workspace_bytes_cached(batch, total_faces, height, width, knum, want)
        else:
            n = _lib.lib().dibr_b200_workspace_bytes(batch, total_faces, height, width)
        if len(_ws_bytes) < 4096:
            _ws_bytes[key] = n
    if n == 0:
        raise RuntimeError("kaolin_b200: unsupported problem size "
                           f"(batch={batch}, faces={total_faces}, image={height}x{width})")
    return torch.empty(n, dtype=torch.uint8, device=device)


def forward(mode, height, width, fvz, fvi, ff, fnz, valid_u8, multiplier, eps,
            sigmainv, boxlen_m, knum, face_idx_in=None):
    """Calls dibr_b200_forward, _bf16 or _f64 (from the dtypes of fvi and ff); returns
    (feat, face_idx, weights, soft, workspace).  Inputs that do not start on a 16-byte boundary are
    copied first (``aligned``).

    float32 / bf16: the barycentric weights are not stored (the third slot is None): the backward
    recomputes them bit for bit from face_idx, the vertices and the same multiplier and eps.
    float64: they are, as (B,H,W,3) doubles for the backward to read; boxlen_m stays a double."""
    dev = fvi.device
    B, F = fvi.shape[0], fvi.shape[1]
    D = 0 if ff is None else ff.shape[-1]
    fvz, fvi, ff, fnz, valid_u8, face_idx_in = map(aligned, (fvz, fvi, ff, fnz, valid_u8, face_idx_in))
    raster = bool(mode & _lib.RASTER)
    soft_on = bool(mode & _lib.SOFT_MASK)
    f64 = fvi.dtype == torch.float64
    bf16 = ff is not None and ff.dtype == torch.bfloat16
    real = torch.float64 if f64 else torch.float32
    feat = torch.empty((B, height, width, D), dtype=torch.bfloat16 if bf16 else real,
                       device=dev) if raster else None
    wts = torch.empty((B, height, width, 3), dtype=real, device=dev) if raster and f64 else None
    idx = torch.empty((B, height, width), dtype=torch.int64, device=dev) if raster else face_idx_in
    soft = torch.empty((B, height, width), dtype=real, device=dev) if soft_on else None
    if B == 0:       # an empty view shard (batch < world size): empty images, nothing to launch
        return feat, idx, wts, soft, None
    ws = workspace(B, B * F, height, width, dev, knum if soft_on else 0, f64)
    name = "dibr_b200_forward_f64" if f64 else "dibr_b200_forward"
    _lib.call(name + "_bf16" if bf16 else name, dev,
              B, F, height, width, D, fvz, fvi, ff, fnz, valid_u8,
              float(multiplier), float(eps), mode, float(sigmainv), float(boxlen_m), int(knum),
              feat, idx, wts, soft, ws, ws.numel(), what=name)
    return feat, idx, wts, soft, ws



def _backward_call(B, F, height, width, D, g_feat, g_soft, face_idx, wts, soft, fvi, ff, multiplier, eps,
                   sigmainv, boxlen_m, knum, g_fvi, g_ff, ws, ws_bytes, flags, dev, views=None):
    bf16 = ff is not None and ff.dtype == torch.bfloat16
    if g_feat is not None and ff is not None and g_feat.dtype != ff.dtype:
        raise RuntimeError(f"dibr_b200_backward: grad_features is {g_feat.dtype}, face_features is {ff.dtype}")
    if views is not None:
        _lib.call("dibr_b200_backward_views", dev,
                  B, F, height, width, D, g_feat, g_soft, face_idx, wts, soft,
                  fvi, ff, int(bf16), float(multiplier), float(eps), float(sigmainv), float(boxlen_m),
                  int(knum), g_fvi, g_ff, ws, ws_bytes, int(flags), int(views[0]), int(views[1]))
        return
    name = "dibr_b200_backward_f64" if fvi.dtype == torch.float64 else "dibr_b200_backward"
    _lib.call(name + "_bf16" if bf16 else name, dev,
              B, F, height, width, D, g_feat, g_soft, face_idx, wts, soft,
              fvi, ff, float(multiplier), float(eps), float(sigmainv), float(boxlen_m),
              int(knum), g_fvi, g_ff, ws, ws_bytes, int(flags), what=name)


def backward(height, width, g_feat, g_soft, face_idx, wts, soft, fvi, ff, multiplier, eps,
             sigmainv, boxlen_m, knum, ws, bins_valid, feature_grad_hook=None, views=None, out=None):
    """Calls dibr_b200_backward, _bf16 or _f64 (from the dtypes of fvi and ff); returns
    (grad_face_vertices_image, grad_face_features in the precision of fvi).

    ``wts`` is None after a float32 / bf16 ``forward`` (the kernels recompute the weights;
    ``multiplier`` and ``eps`` must then be the forward's) or the (B,H,W,3) weights of the same
    forward, which are read (always so in float64).

    ``views=(v0, v1)`` restricts the call to those views of the batch (dibr_b200_backward_views: all
    tensors stay the full-batch ones, only rows v0..v1-1 of the gradients are written) and ``out=
    (g_fvi, g_ff)`` supplies the full-batch gradient buffers to write into - together they let a
    caller pipeline view chunks (kaolin_b200.multi_gpu.pipelined_backward_all_gather).  Both serve
    float32 / bf16 only.  Inputs that do not start on a 16-byte boundary are copied first
    (``aligned``); an ``out=`` buffer that does not raises ValueError.

    ``feature_grad_hook`` (per call — there is no process-global state): called as
    ``hook(g_ff)`` between the two branches of a fused backward.  grad_face_features is
    final after the rasterize branch, so e.g. its all-gather can travel while the
    soft-mask branch runs (kaolin_b200.multi_gpu.OverlappedGradAllGather).  The float64
    backward is one kernel: it calls the hook once, at the end."""
    dev = fvi.device
    B, F = fvi.shape[0], fvi.shape[1]
    D = 0 if ff is None else ff.shape[-1]
    f64 = fvi.dtype == torch.float64
    if f64 and (views is not None or out is not None):
        raise ValueError("kaolin_b200: views= and out= serve the float32 / bfloat16 backward only")
    if out is not None and any(t is not None and t.data_ptr() % 16 for t in out):
        raise ValueError("kaolin_b200: the out= gradient buffers must start on a 16-byte boundary")
    g_feat, g_soft, face_idx, wts, soft, fvi, ff = map(aligned, (g_feat, g_soft, face_idx, wts, soft, fvi, ff))
    # grad_face_features is accumulated (atomics) in the precision of the vertices whatever the
    # storage type of the features: fp32 for fp32 / bf16
    if B * F == 0 and out is None:       # empty mesh: empty gradients, nothing to launch
        return torch.zeros_like(fvi), (torch.zeros(ff.shape, dtype=fvi.dtype, device=dev) if ff is not None else None)
    if out is not None:
        g_fvi, g_ff = out
    else:
        g_fvi = torch.empty_like(fvi)
        g_ff = torch.empty(ff.shape, dtype=fvi.dtype, device=dev) if ff is not None else None
    # The workspace carries forward's bins / hit cache (soft-mask branch, bins_valid) and the
    # per-face records of the row-walk rasterize backward; without forward state a fresh
    # minimum-size one serves both.
    if ws is None:
        ws = workspace(B, B * F, height, width, dev, f64=f64)
        bins_valid = False
    ws_bytes = ws.numel()
    flags = _lib.BINS_VALID if bins_valid else 0
    hook = feature_grad_hook
    both = hook is not None and g_feat is not None and g_soft is not None
    if both and D > 0 and not f64:
        # two calls: rasterize branch (g_ff final -> hook), then the soft-mask branch added on top
        _backward_call(B, F, height, width, D, g_feat, None, face_idx, wts, None, fvi, ff, multiplier, eps,
                       sigmainv, boxlen_m, knum, g_fvi, g_ff, ws, ws_bytes, 0, dev, views)
        hook(g_ff)
        _backward_call(B, F, height, width, D, None, g_soft, face_idx, wts, soft, fvi, ff, multiplier, eps,
                       sigmainv, boxlen_m, knum, g_fvi, None, ws, ws_bytes, flags | _lib.ACCUMULATE, dev, views)
    else:
        _backward_call(B, F, height, width, D, g_feat, g_soft, face_idx, wts, soft, fvi, ff, multiplier, eps,
                       sigmainv, boxlen_m, knum, g_fvi, g_ff, ws, ws_bytes, flags, dev, views)
        if both and f64:
            hook(g_ff)
    return g_fvi, g_ff
