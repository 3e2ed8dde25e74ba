"""The device-to-host pipeline the exporters share (pseudo_gt_export.py, sample_export.py): each batch's GPU work leaves
the bytes to be written in one device staging buffer, ONE copy per batch moves them to a pinned host slot (two slots,
CUDA events), and a thread pool writes the files while the GPU works on the next batch."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

import b3d


def byte_layout(fields):
    """fields: [(name, dtype, shape)] -> ({name: (byte offset, dtype, shape)}, total bytes), every field 16-byte aligned."""
    out, off = {}, 0
    for name, dt, shape in fields:
        out[name] = (off, dt, tuple(shape))
        off += (int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size() + 15) // 16 * 16
    return out, off


def views(buf, layout):
    """The typed views of a uint8 buffer that byte_layout describes."""
    return {k: buf[o:o + int(np.prod(s)) * torch.empty(0, dtype=dt).element_size()].view(dt).view(s)
            for k, (o, dt, s) in layout.items()}


class Staging:
    """One device staging buffer and two pinned host slots of the same size, allocated at the first batch: every batch
    but the last must have the first batch's size, so the first is the largest.  what: the name errors carry."""

    def __init__(self, device, what):
        self.device, self.what = device, what
        self.buffer = self.slots = None

    def device_buffer(self, nbytes, batch_size):
        """The device staging buffer (at least nbytes)."""
        if self.buffer is None:
            self.buffer = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self.slots = [torch.empty(nbytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        if nbytes > self.buffer.numel():
            raise b3d.B3DError(f'{self.what}: a batch of {batch_size} needs {nbytes} staging bytes, '
                               f'{self.buffer.numel()} were allocated for the first batch; only the last batch may be '
                               'smaller')
        return self.buffer

    def run(self, batches, device_batch, drain, writers):
        """device_batch(batch) -> (meta, nbytes, count): enqueues one batch's GPU work, which leaves its bytes in
        device_buffer()[:nbytes]; count is the number of writes its drain will queue.  drain(host, meta, submit): the
        host side of one staged batch, called once its copy has arrived (the only host synchronisation per batch) while
        the GPU works on the next one; host is the pinned slot's first nbytes, submit(fn, *args) queues a write on a
        pool of `writers` threads.  The slot is refilled two batches later, so drain copies out what its writes need.
        At most max(4 writers, 2 count) writes stay queued.  Returns after every write has finished (a failed write
        raises)."""
        events = [None, None]
        pending, futures = None, []
        stream = torch.cuda.current_stream(self.device)
        with ThreadPoolExecutor(max_workers=max(1, int(writers))) as pool:
            def submit(fn, *args):
                futures.append(pool.submit(fn, *args))

            def flush(p):
                slot, meta, nbytes = p
                events[slot].synchronize()
                drain(self.slots[slot][:nbytes], meta, submit)

            try:
                for n, batch in enumerate(batches):
                    # slot n % 2 last held batch n - 2, which flush() handed to drain during iteration n - 1
                    slot = n % 2
                    meta, nbytes, count = device_batch(batch)
                    self.slots[slot][:nbytes].copy_(self.buffer[:nbytes], non_blocking=True)
                    events[slot] = torch.cuda.Event()
                    events[slot].record(stream)
                    if pending is not None:
                        flush(pending)
                    pending = (slot, meta, nbytes)
                    throttle(futures, max(4 * int(writers), 2 * count))
                if pending is not None:
                    flush(pending)
                for f in futures:
                    f.result()                  # a failed write raises here
            finally:
                for f in futures:
                    f.cancel()


def throttle(futures, limit):
    """Keep at most `limit` writes queued: each holds its data in host memory until it is written."""
    while sum(1 for f in futures if not f.done()) > limit:
        next(f for f in futures if not f.done()).result()
