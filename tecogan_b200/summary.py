"""Training observability without TensorFlow: a TensorBoard scalar event writer and the stdout tee of the reference's
main.py (`Logger`, main.py:126-136).

An event file `events.out.tfevents.<unix time>.<hostname>` is a TFRecord stream: per record a little-endian u64 payload
length, the masked CRC32C of those 8 bytes, the payload, the masked CRC32C of the payload.  Each payload is an `Event`
proto (tensorflow/core/util/event.proto): the first carries file_version = "brain.Event:2"; every later one wall_time
(field 1, double), step (2, int64) and a Summary (5) whose repeated Value (1) holds tag (1, string) and simple_value
(2, float) -- what tf.summary.scalar + FileWriter.add_summary write -- or an image (4): Summary.Image with height (1,
int32), width (2), colorspace (3) and encoded_image_string (4), what the reference's GIF summaries write
(lib/ops.py:434-484).  CRC and protobuf encoding are tf_bundle's."""
import os
import socket
import struct
import sys
import time

from .tf_bundle import _field, _pb_bytes, _pb_varint, crc32c, mask_crc


def _record(payload):
    header = struct.pack("<Q", len(payload))
    return (header + struct.pack("<I", mask_crc(crc32c(header))) + payload
            + struct.pack("<I", mask_crc(crc32c(payload))))


def _event(wall_time, step=None, file_version=None, summary=None):
    out = _field(1, 1, struct.pack("<d", wall_time))
    if step is not None:
        out += _pb_varint(2, int(step))
    if file_version is not None:
        out += _pb_bytes(3, file_version.encode())
    if summary is not None:
        out += _pb_bytes(5, summary)
    return out


def _scalar_summary(pairs):
    return b"".join(_pb_bytes(1, _pb_bytes(1, str(tag).encode()) + _field(5, 2, struct.pack("<f", float(v))))
                    for tag, v in pairs)


def _image_summary(items):
    return b"".join(_pb_bytes(1, _pb_bytes(1, str(tag).encode()) + _pb_bytes(4, _pb_varint(1, int(h)) + _pb_varint(2, int(w))
                                                                             + _pb_varint(3, 3) + _pb_bytes(4, bytes(data))))
                    for tag, h, w, data in items)


class EventWriter:
    """Scalar and image summaries for TensorBoard in `logdir` (tf.summary.FileWriter's file naming and record format)."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        self.path = os.path.join(logdir, "events.out.tfevents.%d.%s" % (int(time.time()), socket.gethostname()))
        self._f = open(self.path, "ab")
        self._write(_event(time.time(), step=0, file_version="brain.Event:2"))

    def _write(self, payload):
        self._f.write(_record(payload))
        self._f.flush()               # a running TensorBoard sees every summary as soon as it is written

    def add_scalars(self, step, pairs):
        """One Event at `step` holding a simple_value per (tag, value) of `pairs`."""
        self._write(_event(time.time(), step=step, summary=_scalar_summary(pairs)))

    def add_images(self, step, items):
        """One Event at `step` holding an RGB image (colorspace 3) per (tag, height, width, encoded bytes) of `items`."""
        self._write(_event(time.time(), step=step, summary=_image_summary(items)))

    def close(self):
        self._f.close()


class Tee:
    """sys.stdout replacement that also appends everything printed to a file (reference main.py:126-136)."""

    def __init__(self, path, stream=None):
        self.terminal = stream if stream is not None else sys.stdout
        self.log = open(path, "a")

    def write(self, message):
        self.terminal.write(message)
        self.log.write(message)

    def flush(self):
        self.terminal.flush()
        self.log.flush()

    def __getattr__(self, name):      # isatty, fileno, encoding, ... of the terminal stream
        return getattr(self.terminal, name)

    def close(self):
        self.log.close()
