"""Temporal stabilisation of video (DESIGN.md §3.3.6): each stylised frame is blended with its stabilised predecessor, warped
by the optical flow of the content frames, where the flow is confident:

    O_t(x) = round(P_t(x) + beta c_t(x) (O_{t-1}(x + w_t(x)) - P_t(x)))

The flow, the confidence and the blend run on the device (csrc/flow.cu, through the C ABI); a ``TemporalState`` carries the
previous frame's luminance and stabilised output from one ``predict_batch`` call to the next, so the result does not depend
on how a clip is cut into calls.
"""
from __future__ import annotations

import torch

from . import _capi, options


def _stream():
    return torch.cuda.current_stream().cuda_stream


class TemporalState(object):
    """The temporal state of one clip: ``strength`` (beta, in [0, 1)), the luminance [H, W] of the last frame (at the
    stylised size) and its stabilised uint8 output [H, W, 3], both on the device.  ``reset()`` starts the clip again."""

    def __init__(self, strength):
        self.strength = options.check_temporal_strength(strength)
        self.reset()

    def reset(self):
        self.prev_y = None
        self.prev_out = None


def luminance(frames):
    """uint8 CUDA [N, H, W, 3] -> float32 [N, H, W]."""
    lib = _capi.load()
    Y = torch.empty(frames.shape[:3], dtype=torch.float32, device=frames.device)
    _capi.check(lib.wctb200_luminance_u8(frames.data_ptr(), frames.numel() // 3, Y.data_ptr(), _stream()))
    return Y


def flow_pairs(Y):
    """float32 CUDA [M, H, W], M >= 2 -> flows [2 (M - 1), 2, H, W] (backward, forward for every consecutive pair)."""
    lib = _capi.load()
    M, H, W = Y.shape
    nbytes = lib.wctb200_flow_pairs_workspace_bytes(M, H, W)
    if nbytes == 0:
        raise _capi.WctB200Error("flow_pairs: bad geometry %s" % ((M, H, W),))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=Y.device)
    flows = torch.empty((2 * (M - 1), 2, H, W), dtype=torch.float32, device=Y.device)
    _capi.check(lib.wctb200_flow_pairs(Y.data_ptr(), M, H, W, flows.data_ptr(), ws.data_ptr(), nbytes, _stream()))
    return flows


def confidence(Y, flows):
    """uint8 masks [M - 1, H, W] and int32 counts [M - 1] (confident pixels before the cut rule)."""
    lib = _capi.load()
    M, H, W = Y.shape
    mask = torch.empty((M - 1, H, W), dtype=torch.uint8, device=Y.device)
    counts = torch.empty(M - 1, dtype=torch.int32, device=Y.device)
    _capi.check(lib.wctb200_flow_confidence(Y.data_ptr(), M, H, W, flows.data_ptr(), mask.data_ptr(), counts.data_ptr(),
                                            _stream()))
    return mask, counts


def blend_(frames, prev, flows, masks, beta):
    """The recurrent blend in place on uint8 CUDA frames [N, H, W, 3]; ``prev`` the stabilised frame before frame 0, or None."""
    lib = _capi.load()
    N, H, W = frames.shape[:3]
    _capi.check(lib.wctb200_temporal_blend_u8(frames.data_ptr(), N, H, W, 0 if prev is None else prev.data_ptr(),
                                              flows.data_ptr(), masks.data_ptr(), float(beta), _stream()))
    return frames


def stabilize_(state, contents, frames):
    """Stabilise the stylised uint8 CUDA frames [N, H, W, 3] in place, given the content frames [N, H', W', 3] they were
    stylised from (resized to H x W by the device resize when the sizes differ), and advance ``state``.  A frame whose size
    differs from the state's previous frame starts the clip again."""
    from .device_image import imresize
    H, W = frames.shape[1], frames.shape[2]
    if (contents.shape[1], contents.shape[2]) != (H, W):
        contents = imresize(contents, (H, W))
    Y = luminance(contents.contiguous())
    if state.prev_y is not None and tuple(state.prev_y.shape) == (H, W):
        Ys, prev = torch.cat([state.prev_y[None], Y]), state.prev_out
    else:
        Ys, prev = Y, None
    if Ys.shape[0] >= 2 and state.strength > 0:
        flows = flow_pairs(Ys)
        masks, _ = confidence(Ys, flows)
        blend_(frames, prev, flows, masks, state.strength)
    state.prev_y = Y[-1].clone()
    state.prev_out = frames[-1].clone()
    return frames
