"""Streaming inference recurrence (reference main.py:185-216 graph, main.py:253-268 loop; SURVEY A.9).

State per clip (reference main.py:197-199): pre_inputs (previous LR), pre_gen (previous HR output), pre_warp.
Per frame i:   i > 0:  flow = fnet(pre_inputs ++ LR_i);  pre_warp = warp(pre_gen, upscale_four(4*pad_sym(flow)))
               HR_i = generator_F(LR_i ++ space_to_depth(pre_warp));  pre_inputs = LR_i;  pre_gen = deprocess(HR_i)
frame 0 uses pre_warp = 0.

bf16 mode keeps everything in pre-allocated device buffers and replays ONE CUDA graph per frame
(~57 wgmma launches + warp/s2d + resample kernels); fp32 mode runs the differentiable mirror under no_grad.

Look-ahead (bf16 mode, step(lr, next_lr=...) / run_sequence): the flow of frame i+1 depends only on LR_i and LR_{i+1}
(main.py:211), not on any HR output, so fnet(LR_i ++ LR_{i+1}) is captured on a second stream of the frame graph and
runs concurrently with generator_F of frame i; frame i+1 then starts directly with warp + generator.  Same kernels on
the same inputs in the same order per buffer, hence bit-identical outputs to the serial recurrence (tested).
"""
import torch

from . import config
from . import kernels as K
from ._ffi import call, ptr, stream_ptr
from .tc_nets import (FNetPlan, GeneratorPlan, LR_OFF, S2D_OFF, _ensure_vars_fnet, _ensure_vars_generator,
                      _f32_slice_to_bf16)
from .variables import default_store, variable_scope

f32 = torch.float32
bf16 = torch.bfloat16


class InferenceEngine:
    """B independent clips of LR size h x w streamed frame by frame."""

    def __init__(self, h, w, num_resblock=16, batch=1, use_graph=True, device="cuda"):
        if h < 8 or w < 8:
            raise ValueError("InferenceEngine: LR frames must be at least 8x8")
        self.h, self.w, self.B, self.nrb = h, w, batch, num_resblock
        self.device = torch.device(device)
        self.precision = config.precision()
        self.use_graph = use_graph and self.precision == "bf16"
        self.lr_in = torch.zeros((batch, h, w, 3), device=self.device, dtype=f32)     # static input buffer
        self.prev_lr = torch.zeros_like(self.lr_in)
        self.out01 = torch.zeros((batch, 4 * h, 4 * w, 3), device=self.device, dtype=f32)
        self.out_u8 = torch.zeros((batch, 4 * h, 4 * w, 3), device=self.device, dtype=torch.uint8)
        self.frame_idx = 0
        self.graph = None
        self.graph_la = None          # frame graph with the next frame's fnet on a second stream
        self.graph_tail = None        # frame graph that consumes a precomputed flow, no look-ahead
        self.flow_ready = False       # self.flow_cur holds fnet(prev_lr ++ lr_in) for the frame about to be processed
        self.launches_per_frame = 0
        if self.precision == "bf16":
            with variable_scope('generator'), variable_scope('generator_unit') as gs:
                _ensure_vars_generator(num_resblock)
                self.gen = GeneratorPlan(gs, batch, h, w, num_resblock, self.device)
            with variable_scope('fnet'), variable_scope('autoencode_unit') as fs:
                _ensure_vars_fnet()
                self.fnet = FNetPlan(fs, batch, h, w, self.device)
            self.launches_per_frame = self.gen.launches + self.fnet.launches + 5
            self.lr_next = torch.zeros_like(self.lr_in)
            self.flow_cur = torch.zeros_like(self.fnet.flow)
            self._side = torch.cuda.Stream(device=self.device)
            # the generator chain is the critical path of a frame: its kernel nodes get the higher stream priority, the
            # look-ahead fnet fills the SMs it leaves idle
            self._crit = torch.cuda.Stream(device=self.device, priority=-1)
        else:
            self.pre_gen = torch.zeros((batch, 4 * h, 4 * w, 3), device=self.device, dtype=f32)
            self.pre_warp = torch.zeros_like(self.pre_gen)

    # ------------------------------------------------------------------ bf16 / wgmma path
    def _frame_first(self):
        self.gen.x_in[..., S2D_OFF:S2D_OFF + 48].zero_()
        _f32_slice_to_bf16(self.lr_in, 0, 3, self.gen.x_in, LR_OFF)
        self.gen.run(self.lr_in, 3)
        self._finish()

    def _frame_next(self):
        g, f = self.gen, self.fnet
        _f32_slice_to_bf16(self.prev_lr, 0, 3, f.x_in, 0)
        _f32_slice_to_bf16(self.lr_in, 0, 3, f.x_in, 3)
        flow_lr = f.run()
        # fused: symmetric pad + x4 + upscale_four + warp(previous output, read as [-1,1] and deprocessed) + s2d
        K.warp_s2d_fused(g.out, flow_lr, g.x_in, S2D_OFF, in_scale=0.5, in_shift=0.5)
        _f32_slice_to_bf16(self.lr_in, 0, 3, g.x_in, LR_OFF)
        g.run(self.lr_in, 3)
        self._finish()

    def _finish(self, keep_lr=True):
        n = self.out01.numel()
        call("teco_deprocess_u8", ptr(self.gen.out, f32), ptr(self.out01, f32), ptr(self.out_u8, torch.uint8), n, stream_ptr())
        if keep_lr:
            self.prev_lr.copy_(self.lr_in)

    # -- look-ahead pieces
    def _fnet_ahead(self):
        """fnet(LR_i ++ LR_{i+1}) from lr_in / lr_next into self.fnet.flow (current stream)."""
        f = self.fnet
        _f32_slice_to_bf16(self.lr_in, 0, 3, f.x_in, 0)
        _f32_slice_to_bf16(self.lr_next, 0, 3, f.x_in, 3)
        f.run()

    def _gen_from_flow(self, after_warp=None, lr_ready=None):
        g = self.gen
        K.warp_s2d_fused(g.out, self.flow_cur, g.x_in, S2D_OFF, in_scale=0.5, in_shift=0.5)
        if after_warp is not None:
            after_warp.record()
        if lr_ready is None:
            _f32_slice_to_bf16(self.lr_in, 0, 3, g.x_in, LR_OFF)
        else:
            torch.cuda.current_stream().wait_event(lr_ready)   # LR channels of x_in and bicubic(LR) came from the side stream
        g.run(self.lr_in, 3, bicubic=lr_ready is None)
        self._finish(keep_lr=False)

    def _frame_lookahead(self):
        """Frame i from the precomputed flow on the current stream; fnet for frame i+1 on the side stream."""
        main, side = torch.cuda.current_stream(), self._side
        warped, lr_ready = torch.cuda.Event(), torch.cuda.Event()
        side.wait_stream(main)                       # fork
        with torch.cuda.stream(side):
            # the LR-only parts of this frame's generator leave the critical path too (disjoint channels of x_in
            # from the warp's space-to-depth channels)
            _f32_slice_to_bf16(self.lr_in, 0, 3, self.gen.x_in, LR_OFF)
            self.gen.run_bicubic(self.lr_in, 3)
            lr_ready.record()
            self._fnet_ahead()
        self._gen_from_flow(after_warp=warped, lr_ready=lr_ready)
        with torch.cuda.stream(side):
            side.wait_event(warped)                  # flow_cur has been consumed by this frame's warp
            self.flow_cur.copy_(self.fnet.flow)
        main.wait_stream(side)                       # join
        self.prev_lr.copy_(self.lr_in)
        self.lr_in.copy_(self.lr_next)

    def _frame_tail(self):
        self._gen_from_flow()
        self.prev_lr.copy_(self.lr_in)

    # ------------------------------------------------------------------ fp32 path (exact-parity mode)
    def _frame_fp32(self):
        from .lib.frvsr import fnet, generator_F
        from .lib.ops import deprocess

        class _F:
            num_resblock = self.nrb
        h, w = self.h, self.w
        with torch.no_grad():
            cur = self.lr_in
            if self.frame_idx > 0:
                with variable_scope('fnet'):
                    flow_lr = fnet(torch.cat((self.prev_lr, cur), dim=-1), reuse=self.frame_idx > 1)
                # tf.pad SYMMETRIC + *4 + upscale_four + dense_image_warp + space_to_depth, fused (main.py:212-215,201)
                s2d = torch.zeros((self.B, h, w, 48), device=self.device, dtype=f32)
                K.warp_s2d_fused(self.pre_gen, flow_lr, s2d, 0, warped_out=self.pre_warp)
            else:
                s2d = torch.zeros((self.B, h, w, 48), device=self.device, dtype=f32)
            with variable_scope('generator'):
                gen_out = generator_F(torch.cat((cur, s2d), dim=-1), 3, reuse=self.frame_idx > 0, FLAGS=_F)
            self.pre_gen = deprocess(gen_out)
            self.out01.copy_(self.pre_gen)
            call("teco_to_u8", ptr(self.out01, f32), ptr(self.out_u8, torch.uint8), self.out01.numel(), stream_ptr())
            self.prev_lr.copy_(cur)

    # ------------------------------------------------------------------ public API
    def reset(self):
        self.frame_idx = 0
        self.flow_ready = False

    def _check_frame(self, lr, what):
        if lr.dim() == 3:
            lr = lr.unsqueeze(0)
        if tuple(lr.shape) != tuple(self.lr_in.shape):
            raise ValueError("InferenceEngine.step: expected %s of shape %s, got %s"
                             % (what, tuple(self.lr_in.shape), tuple(lr.shape)))
        return lr

    def step(self, lr=None, next_lr=None):
        """Advance one frame.  lr: [B,h,w,3] (or [h,w,3] when B == 1) fp32 in [0,1], CUDA or pinned host; if None the
        caller has already filled self.lr_in.  Returns self.out01 ([B,4h,4w,3] fp32 in [0,1], overwritten each step).

        next_lr (bf16 mode): the FOLLOWING LR frame.  When given, its flow is computed concurrently with this frame's
        generator, and the next call starts from that flow; the next call's `lr` must then be this `next_lr` (it is
        already on the device and is not uploaded again)."""
        if next_lr is not None and self.precision != "bf16":
            next_lr = None                       # the fp32 exact-parity mode stays strictly serial
        pending = self.flow_ready
        if lr is not None and not pending:
            self.lr_in.copy_(self._check_frame(lr, "LR frame"), non_blocking=True)
        if next_lr is not None:
            self.lr_next.copy_(self._check_frame(next_lr, "next LR frame"), non_blocking=True)
        if self.precision != "bf16":
            self._frame_fp32()
        elif self.frame_idx == 0 or (next_lr is not None and not pending):
            # first frame of a clip (or look-ahead requested without a pending flow): serial frame, then prime the flow
            if self.frame_idx == 0:
                self._frame_first()
            else:
                self._frame_next()
            if next_lr is not None:
                self._fnet_ahead()
                self.flow_cur.copy_(self.fnet.flow)
                self.lr_in.copy_(self.lr_next)
                self.flow_ready = True
        elif pending:
            body = self._frame_lookahead if next_lr is not None else self._frame_tail
            if not self.use_graph:
                body()
            else:
                attr = "graph_la" if next_lr is not None else "graph_tail"
                if getattr(self, attr) is None:
                    setattr(self, attr, self._capture(body))
                getattr(self, attr).replay()
            self.flow_ready = next_lr is not None
        elif not self.use_graph:
            self._frame_next()
        else:
            if self.graph is None:
                self.graph = self._capture(self._frame_next)
            self.graph.replay()
        self.frame_idx += 1
        return self.out01

    def _capture(self, body):
        # warm-up once eagerly on a side stream (sets function attributes, builds tensor maps), then capture;
        # the recurrent state is restored after both passes so that the replay sees the real previous frame
        state = (self.gen.out, self.prev_lr, self.gen.x_in, self.lr_in, self.lr_next, self.flow_cur, self.fnet.flow)
        snap = [t.clone() for t in state]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            body()
        torch.cuda.current_stream().wait_stream(s)
        for t, v in zip(state, snap):
            t.copy_(v)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        # thread-local capture: the streaming command's reader and writer threads keep decoding, copying and
        # synchronising their own streams while this thread captures (main.py::super_resolve_frames)
        with torch.cuda.graph(graph, stream=self._crit, capture_error_mode="thread_local"):
            body()
        for t, v in zip(state, snap):
            t.copy_(v)
        return graph

    def run_sequence(self, frames, out="f32", lookahead=True):
        """frames: iterable of [h,w,3] / [B,h,w,3] tensors.  Returns a list of CUDA tensors, one per frame
        ('f32': [0,1] floats; 'u8': save_img quantisation, reference lib/ops.py:521-523)."""
        self.reset()
        res = []
        frames = list(frames)
        for i, fr in enumerate(frames):
            nxt = frames[i + 1] if (lookahead and i + 1 < len(frames)) else None
            self.step(fr, next_lr=nxt)
            res.append((self.out01 if out == "f32" else self.out_u8).clone())
        return res


class ClipEngine:
    """B independent clips of T frames each (LR h x w), advanced in lock-step: the metric's workload ("10-frame clips",
    BASELINE.json) and the shape of the reference's training recurrence (lib/Teco.py:102-164) used for inference.

    All LR frames of a clip are known up front, so -- exactly as lib/Teco.py:102-117 does -- the flow of every
    consecutive pair is estimated first (it depends on LR frames only, main.py:211); the generator recurrence
    (main.py:212-216 per frame) then runs frame by frame with the batch of B clips as the GEMM M dimension.  The whole
    clip batch is ONE CUDA graph replay; frame 0 of every clip starts from pre_warp = 0 (main.py:199).

    run(lr_clip): lr_clip [T,B,h,w,3] fp32 in [0,1] (CUDA or pinned host, time-major so that a frame of all clips is one
    contiguous block) -> self.clip_u8 [T,B,4h,4w,3] uint8 (save_img quantisation, lib/ops.py:521-523); the fp32 output of
    the last frame stays in self.out01."""

    def __init__(self, h, w, T, num_resblock=16, batch=1, use_graph=True, device="cuda"):
        """FNet runs once per clip batch, over all B * (T - 1) consecutive frame pairs (they are independent, and
        lib/Teco.py:102-117 batches them all too): fewer, fuller launches.  Every FNet convolution computes each output in a
        fixed order whatever the batch size, so the flows are byte-identical to one-pair passes over the same frames."""
        if h < 8 or w < 8:
            raise ValueError("ClipEngine: LR frames must be at least 8x8")
        if T < 1:
            raise ValueError("ClipEngine: a clip has at least one frame")
        if config.precision() != "bf16":
            raise ValueError("ClipEngine runs the wgmma path; use InferenceEngine for the fp32 exact-parity mode")
        self.h, self.w, self.T, self.B, self.nrb = h, w, T, batch, num_resblock
        self.device = torch.device(device)
        self.use_graph = use_graph
        self.clip_in = torch.zeros((T, batch, h, w, 3), device=self.device, dtype=f32)
        self.clip_u8 = torch.zeros((T, batch, 4 * h, 4 * w, 3), device=self.device, dtype=torch.uint8)
        self.out01 = torch.zeros((batch, 4 * h, 4 * w, 3), device=self.device, dtype=f32)
        with variable_scope('generator'), variable_scope('generator_unit') as gs:
            _ensure_vars_generator(num_resblock)
            self.gen = GeneratorPlan(gs, batch, h, w, num_resblock, self.device)
        with variable_scope('fnet'), variable_scope('autoencode_unit') as fs:
            _ensure_vars_fnet()
            # pair (t - 1, t) of clip b is FNet image (t - 1) * B + b: time-major, so frames 0 .. T-2 and 1 .. T-1 of all
            # clips are two contiguous blocks of clip_in, and the flows land in self.flows[t - 1][b]
            self.fnet = FNetPlan(fs, batch * max(T - 1, 1), h, w, self.device)
        self.flows = self.fnet.flow.view((max(T - 1, 1), batch) + tuple(self.fnet.flow.shape[1:]))
        self.graph = None
        # our kernel launches per clip batch: one fnet pass, then per frame warp/pack/generator/deprocess
        self.launches = (self.fnet.launches + 2 if T > 1 else 0) + T * (self.gen.launches + 2) + (T - 1)

    def _body(self):
        g, f, T = self.gen, self.fnet, self.T
        hw3 = (self.h, self.w, 3)
        if T > 1:
            _f32_slice_to_bf16(self.clip_in[:T - 1].view(-1, *hw3), 0, 3, f.x_in, 0)
            _f32_slice_to_bf16(self.clip_in[1:].view(-1, *hw3), 0, 3, f.x_in, 3)
            f.run()
        n = self.out01.numel()
        for t in range(T):
            if t == 0:
                g.x_in[..., S2D_OFF:S2D_OFF + 48].zero_()
            else:
                K.warp_s2d_fused(g.out, self.flows[t - 1], g.x_in, S2D_OFF, in_scale=0.5, in_shift=0.5)
            _f32_slice_to_bf16(self.clip_in[t], 0, 3, g.x_in, LR_OFF)
            g.run(self.clip_in[t], 3)
            call("teco_deprocess_u8", ptr(g.out, f32), ptr(self.out01 if t == T - 1 else None, f32), ptr(self.clip_u8[t], torch.uint8), n, stream_ptr())

    def replay(self):
        """Process the clip batch already in self.clip_in."""
        if not self.use_graph:
            self._body()
            return self.clip_u8
        if self.graph is None:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._body()                      # eager warm-up (function attributes, allocator)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._body()
        self.graph.replay()
        return self.clip_u8

    def run(self, lr_clip):
        if tuple(lr_clip.shape) != tuple(self.clip_in.shape):
            raise ValueError("ClipEngine.run: expected LR clips of shape %s (time-major), got %s"
                             % (tuple(self.clip_in.shape), tuple(lr_clip.shape)))
        self.clip_in.copy_(lr_clip, non_blocking=True)
        return self.replay()
