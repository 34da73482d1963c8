"""Write-behind of uint8 device frames to image files, shared by the inference command (main.py::super_resolve_frames)
and the training-data preparation (tecogan_b200/data_prepare.py)."""

WRITE_SLOTS = 3           # output frames between the producer and the files: encoding, copied back, being written


class FrameWriter:
    """The write-behind half of super_resolve_frames and data_prepare.  put(out_u8, path) copies a uint8 [h, w, 3] RGB
    device frame into a free slot of a small ring on the current (the producer's) stream -- a frame of another size is
    resized into the slot instead (kernels.resize_lanczos4, cv2's INTER_LANCZOS4: `main.py --outscale`) -- then starts
    its encode -- on the slot's own stream, after an event, with the slot's own encoder buffers -- or, for a format cv2
    writes, the copy back to the host.  Either way the frame is read on the producer's stream, before its next step can
    overwrite it.  One writer thread takes the slots in order, waits for each, writes its file (lib/ops.py::write_image,
    the rule save_img follows) and hands the slot back; put() waits for a slot whose file is written.  An exception on
    the writer thread is raised by the next put() and by close(); close() joins the thread on every exit.

    With a `sink` (tecogan_b200/y4m.py::Y4MWriter, `main.py --output_y4m`) the frames go to one video stream instead of
    files: put(out_u8) fills the slot as above, converts it on the slot's stream to I420 (kernels.rgb_to_i420, cv2's
    COLOR_RGB2YUV_I420) in the slot's device buffer and copies that back to a pinned host buffer; the writer thread
    appends the frames to the sink in order.  A failed write is raised, unlike a failed image file."""

    def __init__(self, h, w, device, sink=None):
        import queue
        import threading
        import types
        import torch
        self.h, self.w, self.device, self.sink = h, w, torch.device(device), sink
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.jobs, self.free = queue.Queue(), queue.Queue()
        self.error = None
        self.slots = [types.SimpleNamespace(u8=torch.empty((h, w, 3), dtype=torch.uint8, device=self.device),
                                            stream=torch.cuda.Stream(device=self.device), encoders={}, host=None,
                                            i420=None)
                      for _ in range(WRITE_SLOTS)]
        for s in self.slots:
            self.free.put(s)
        self.thread = threading.Thread(target=self._run, name='FrameWriter', daemon=True)
        self.thread.start()

    def put(self, out_u8, path=None):
        import torch
        from tecogan_b200 import kernels as K
        from tecogan_b200.lib import ops
        codec = 'y4m' if self.sink is not None else ops.image_codec(path, self.h, self.w)
        slot = self.free.get()
        if isinstance(slot, BaseException):
            raise slot
        if tuple(out_u8.shape[:2]) == (self.h, self.w):
            slot.u8.copy_(out_u8)
        else:
            K.resize_lanczos4(out_u8, slot.u8)
        ready = torch.cuda.Event()
        ready.record()
        with torch.cuda.stream(slot.stream):
            slot.stream.wait_event(ready)
            if codec == 'y4m':
                if slot.i420 is None:
                    slot.i420 = torch.empty((3 * self.h // 2, self.w), dtype=torch.uint8, device=self.device)
                    slot.host = torch.empty(slot.i420.shape, dtype=torch.uint8, pin_memory=True)
                K.rgb_to_i420(slot.u8, slot.i420)
                slot.host.copy_(slot.i420, non_blocking=True)
                job = None
            elif codec == 'cv2':
                if slot.host is None:
                    slot.host = torch.empty(slot.u8.shape, dtype=torch.uint8, pin_memory=True)
                slot.host.copy_(slot.u8, non_blocking=True)
                job = None
            else:
                if codec not in slot.encoders:
                    slot.encoders[codec] = ops.device_encoder(codec)
                job = slot.encoders[codec].launch(slot.u8, (self.h, self.w))
        self.jobs.put((path, codec, slot, job))

    def _run(self):
        import torch
        from tecogan_b200 import _encode
        from tecogan_b200.lib import ops
        try:
            torch.cuda.set_device(self.device)
            while True:
                item = self.jobs.get()
                if item is None:
                    return
                path, codec, slot, job = item
                if job is None:
                    slot.stream.synchronize()
                    data = slot.host.numpy()
                else:
                    data = _encode.collect([job])[0][0]
                if codec == 'y4m':
                    self.sink.write(data)
                else:
                    ops.write_image(path, codec, data)
                self.free.put(slot)
        except BaseException as e:
            self.error = e
            self.free.put(e)                   # wakes a put() waiting for a slot

    def close(self):
        """Write what is queued (unless the writer failed), join the thread and wait for every slot's stream."""
        self.jobs.put(None)
        self.thread.join()
        for s in self.slots:
            s.stream.synchronize()
