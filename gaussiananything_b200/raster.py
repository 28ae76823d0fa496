"""Batched surfel rasterisation: torch plumbing over the C ABI.

One call renders every (batch item, view) pair -- the whole double loop of
/root/reference/nsr/gs_surfel.py:65-176 -- with one launch set.  Tensors are
only used for device memory, the current stream and autograd bookkeeping; all
arithmetic happens in libga_b200.so.
"""
import ctypes as C

import torch

from . import _lib

_capacity_hint = {}


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


LIST_K = 32          # per-pixel contribution-list capacity used when the caller will ask for gradients


def layout(batch, P, views, H, W, max_instances, list_k=0):
    L = _lib.GaRasterLayout()
    _lib.check(_lib.lib().ga_raster_layout_ex(batch, P, views, H, W, max_instances, int(list_k), C.byref(L)),
               "ga_raster_layout_ex")
    return L


def tile_replicas():
    """Counter replicas per tile in the workspace (GA_TILE_REPLICAS of the library build), read from the layout: with
    64 tiles the counter region, R + 1 words per tile (the counters and the big-tile list), is a whole number of 256-byte
    alignment units."""
    L = layout(1, 1, 1, 128, 128, 1)
    return (L.tile_start - L.tile_count) // (64 * 4) - 1


def workspace_views(ws, L, batch, P, views, H, W, max_instances, list_k=0):
    """Typed views of the workspace sections (for tests / debugging).  The list sections (lists, n_list, tile_flag)
    exist only when the forward ran with list_k > 0; inst_cnt is written only then.  big_tiles holds status[3]
    valid entries."""
    NV, T, HW = batch * views, ((W + 15) // 16) * ((H + 15) // 16), H * W

    def sec(off, dtype, n):
        esz = torch.empty(0, dtype=dtype).element_size()
        return ws[off:off + n * esz].view(dtype)
    lists = {}
    if list_k:
        lists = dict(lists=sec(L.lists, torch.int32, NV * T * list_k * 256 * 4).view(NV * T, list_k, 256, 4),
                     n_list=sec(L.n_list, torch.int32, NV * HW).view(NV, H, W),
                     tile_flag=sec(L.tile_flag, torch.int32, NV * T))
    return dict(
        lists,
        big_tiles=sec(L.tile_count + NV * T * tile_replicas() * 4, torch.int32, NV * T),    # after the tile counters
        inst_cnt=sec(L.inst_cnt, torch.int32, max_instances),
        status=sec(L.status, torch.int32, 16),
        rec=sec(L.rec, torch.float32, NV * P * 24).view(NV, P, 24),
        depth=sec(L.depth, torch.float32, NV * P).view(NV, P),
        rect=sec(L.rect, torch.int32, NV * P).view(NV, P),
        tile_start=sec(L.tile_start, torch.int32, NV * T + 1),
        keys=sec(L.keys, torch.int64, max_instances),
        ids=sec(L.ids, torch.int32, max_instances),
        final_T=sec(L.final_T, torch.float32, NV * 3 * HW).view(NV, 3, H, W),
        n_contrib=sec(L.n_contrib, torch.int32, NV * 2 * HW).view(NV, 2, H, W),
    )


_status_slots = {}


def _status_slot(dev):
    """Pinned 4-int buffer + event for the overlapped status read-back of ga_raster_forward_ex."""
    # one slot per (device, stream): calls on different streams may overlap on the host
    key = (dev.index if dev.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(dev).cuda_stream)
    slot = _status_slots.get(key)
    if slot is None:
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))          # materialises the underlying cudaEvent_t
        slot = (torch.zeros(4, dtype=torch.int32).pin_memory(), ev)
        _status_slots[key] = slot
    return slot


def forward_raw(gauss13, viewmats, projmats, bg, H, W, scale_modifier=1.0, max_instances=None, list_k=None):
    """gauss13 [B,P,13], viewmats/projmats [B,V,4,4] (reference layout), bg [3].
    Returns (color [B,V,3,H,W], allmap [B,V,7,H,W], radii [B,V,P], state).
    list_k: per-pixel contribution lists for the backward (default: LIST_K when gauss13 requires grad, else 0)."""
    if list_k is None:
        list_k = LIST_K if gauss13.requires_grad else 0
    lib = _lib.lib()
    if not gauss13.is_cuda:
        raise RuntimeError("gaussiananything_b200 rasteriser needs CUDA tensors (no CPU fallback)")
    dev = gauss13.device
    B, P, c = gauss13.shape
    assert c == 13
    V = viewmats.shape[1]
    gauss13 = gauss13.contiguous().float()
    viewmats = viewmats.reshape(B * V, 16).contiguous().float()
    projmats = projmats.reshape(B * V, 16).contiguous().float()
    bg = bg.to(device=dev, dtype=torch.float32).contiguous()
    with torch.cuda.device(dev):           # launches go to the tensors' device, not the process's current one
        return _forward_on_device(lib, dev, gauss13, viewmats, projmats, bg, B, P, V, H, W, scale_modifier, max_instances,
                                  int(list_k))


def _forward_on_device(lib, dev, gauss13, viewmats, projmats, bg, B, P, V, H, W, scale_modifier, max_instances, list_k):
    key = (B, P, V, H, W)
    if max_instances is None:
        max_instances = _capacity_hint.get(key, 4 * B * V * P + 1024)
    color = torch.empty(B, V, 3, H, W, device=dev, dtype=torch.float32)
    allmap = torch.empty(B, V, 7, H, W, device=dev, dtype=torch.float32)
    radii = torch.empty(B, V, P, device=dev, dtype=torch.int32)
    host_status, ev = _status_slot(dev)
    while True:
        L = layout(B, P, V, H, W, max_instances, list_k)
        ws = torch.empty(L.total_bytes, device=dev, dtype=torch.uint8)
        # the whole forward is enqueued in one call; the instance count / overflow flag (where upstream reads
        # num_rendered back) is copied to pinned memory right after the tile scan, so this wait returns while the
        # GPU is still scattering, sorting and compositing -- no bubble in the stream
        _lib.check(lib.ga_raster_forward_ex(
            _ptr(gauss13), B, P, V, _ptr(viewmats), _ptr(projmats), _ptr(bg), H, W, float(scale_modifier),
            _ptr(color), _ptr(allmap), _ptr(radii), _ptr(ws), L.total_bytes, max_instances, list_k,
            C.c_void_p(host_status.data_ptr()), C.c_void_p(ev.cuda_event), _stream(dev)),
            "ga_raster_forward_ex")
        ev.synchronize()
        status = host_status.clone()
        if int(status[1]) == 0:
            break
        max_instances = int(int(status[0]) * 1.25) + 1024
        _capacity_hint[key] = max_instances
    state = dict(ws=ws, L=L, max_instances=max_instances, num_rendered=int(status[0]), list_k=list_k,
                 gauss13=gauss13, viewmats=viewmats, projmats=projmats, bg=bg,
                 dims=(B, P, V, H, W), scale_modifier=float(scale_modifier), radii=radii)
    return color, allmap, radii, state


_scratch_pool = {}


def _take_scratch(dev, nbytes):
    """The backward's scratch (the gradient accumulators, 43 MB at 100k surfels x 6 views) is only live inside one
    backward call, so it is kept per (device, stream, size) instead of going through the caching allocator every
    step: large blocks allocated and freed alternately make the allocator split / re-grow its segments, i.e. an
    occasional synchronising cudaMalloc in the middle of a training step."""
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream, nbytes)
    pool = _scratch_pool.setdefault(key, [])
    return key, (pool.pop() if pool else torch.empty(nbytes, device=dev, dtype=torch.uint8))


def backward_raw(state, grad_color, grad_allmap):
    lib = _lib.lib()
    B, P, V, H, W = state["dims"]
    dev = state["gauss13"].device
    grad_color = grad_color.contiguous().float()
    grad_allmap = grad_allmap.contiguous().float()
    nbytes = lib.ga_raster_backward_scratch_bytes(B, P, V)
    with torch.cuda.device(dev):
        pool_key, scratch = _take_scratch(dev, nbytes)
        grad = torch.empty(B, P, 13, device=dev, dtype=torch.float32)
        rc = lib.ga_raster_backward_ex(_ptr(state["gauss13"]), B, P, V, _ptr(state["viewmats"]),
                                    _ptr(state["projmats"]), _ptr(state["bg"]), H, W,
                                    state["scale_modifier"], _ptr(state["radii"]),
                                    _ptr(grad_color), _ptr(grad_allmap),
                                    _ptr(state["ws"]), state["L"].total_bytes, state["max_instances"], state.get("list_k", 0),
                                    _ptr(scratch), nbytes, _ptr(grad), _stream(dev))
    if len(_scratch_pool[pool_key]) < 2:
        _scratch_pool[pool_key].append(scratch)          # reused by later calls on the same stream: stream-ordered, safe
    _lib.check(rc, "ga_raster_backward_ex")
    return grad


class _RasterizeSurfelsBatched(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gauss13, viewmats, projmats, bg, H, W, scale_modifier):
        color, allmap, radii, state = forward_raw(gauss13, viewmats, projmats, bg, H, W, scale_modifier,
                                                  list_k=LIST_K if ctx.needs_input_grad[0] else 0)
        # the tensors the backward re-reads go through save_for_backward, so an in-place change between forward
        # and backward is detected by autograd's version check instead of silently giving wrong gradients
        ctx.save_for_backward(state.pop("gauss13"), state.pop("viewmats"), state.pop("projmats"))
        ctx.state = state
        ctx.mark_non_differentiable(radii)
        return color, allmap, radii

    @staticmethod
    def backward(ctx, grad_color, grad_allmap, _grad_radii):
        g13, vm, pm = ctx.saved_tensors
        grad = backward_raw(dict(ctx.state, gauss13=g13, viewmats=vm, projmats=pm), grad_color, grad_allmap)
        return grad, None, None, None, None, None, None


def rasterize_surfels_batched(gauss13, viewmats, projmats, bg, H, W, scale_modifier=1.0):
    """Differentiable batched rasterisation (grad w.r.t. gauss13 only, like the
    reference, whose cameras and background carry no gradient)."""
    return _RasterizeSurfelsBatched.apply(gauss13, viewmats, projmats, bg, H, W, scale_modifier)


class _RenderPost(torch.autograd.Function):
    """Fused per-view post-processing (reference nsr/gs_surfel.py:121-163) with its own backward kernel."""

    @staticmethod
    def forward(ctx, color, allmap, viewmats):
        lib = _lib.lib()
        B, V, _, H, W = color.shape
        dev = color.device
        color, allmap = color.contiguous(), allmap.contiguous()
        vm = viewmats.reshape(B * V, 16).contiguous().float()
        image = torch.empty(B, V, 3, H, W, device=dev)
        alpha = torch.empty(B, V, 1, H, W, device=dev)
        depth = torch.empty(B, V, 1, H, W, device=dev)
        normal = torch.empty(B, V, 3, H, W, device=dev)
        dist = torch.empty(B, V, 1, H, W, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.ga_render_post_forward(_ptr(color), _ptr(allmap), _ptr(vm), B * V, H, W, _ptr(image),
                                                  _ptr(alpha), _ptr(depth), _ptr(normal), _ptr(dist), _stream(dev)),
                       "ga_render_post_forward")
        ctx.save_for_backward(color, allmap, vm)
        return image, alpha, depth, normal, dist

    @staticmethod
    def backward(ctx, g_image, g_alpha, g_depth, g_normal, g_dist):
        lib = _lib.lib()
        color, allmap, vm = ctx.saved_tensors
        B, V, _, H, W = color.shape
        dev = color.device
        gs = [None if g is None else g.contiguous().float() for g in (g_image, g_alpha, g_depth, g_normal, g_dist)]
        g_color = torch.empty_like(color)
        g_allmap = torch.empty_like(allmap)
        null = C.c_void_p(0)
        ptrs = [null if g is None else _ptr(g) for g in gs]
        with torch.cuda.device(dev):
            _lib.check(lib.ga_render_post_backward(_ptr(color), _ptr(allmap), _ptr(vm), B * V, H, W, *ptrs, _ptr(g_color),
                                                   _ptr(g_allmap), _stream(dev)), "ga_render_post_backward")
        return g_color, g_allmap, None


def render_postprocess(color, allmap, viewmats):
    """(image, alpha, depth, rend_normal, dist) from the raw rasteriser outputs, differentiable."""
    return _RenderPost.apply(color, allmap, viewmats)
