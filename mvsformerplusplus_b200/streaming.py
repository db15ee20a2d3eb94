"""Host-side staging for the hot path: pinned host batches are uploaded on a copy stream into one of a few resident
device slots while the previous batches are still being computed, so the PCIe transfer of the FPN pyramids (531 MB per
DTU reference view) overlaps the kernels instead of preceding them.

Off by default: with `lanes` > 1 consecutive batches run on alternating compute streams (reference views are
independent, SURVEY.md 8e), so that two depth maps in flight can fill the SMs that the latency-bound kernels of one map
(token linears, FMT, U-Net layers) leave idle.

The reference's test loop uploads synchronously (`sample_cuda = tocuda(sample)` then `model.forward(...)`,
test.py / base trainer); this is the drop-in equivalent for a caller that already holds the feature pyramids on the
host.  Only streams, events and `Tensor.copy_` are used here - no computation."""
import torch


class PrefetchingRunner:
    def __init__(self, net, device, slots=2, lanes=1):
        self.net = net
        self.device = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        # compute lanes: lanes == 1 runs on the caller's current stream (as before); otherwise private streams, round-robin
        self.lanes = [torch.cuda.Stream(device=self.device) for _ in range(lanes)] if lanes > 1 else []
        for lane in self.lanes:   # the weights were placed by the caller's stream; nothing else a lane reads comes from it
            lane.wait_stream(torch.cuda.current_stream(self.device))
        self._lane = 0
        self.slots = [dict(bufs=None, ready=torch.cuda.Event(), free=torch.cuda.Event(), tag=None, batch=None)
                      for _ in range(slots)]
        self._next = 0

    # a batch is (features: dict[str, Tensor], proj_matrices: dict[str, Tensor], depth_values: Tensor), pinned host tensors,
    # run by net.forward_features; or (imgs: Tensor [B,V,3,H,W], proj_matrices, depth_values), run by net.forward (a
    # DINOv2MVSNet: images to depth maps, what the reference's test loop uploads)
    @staticmethod
    def _flat(batch):
        f, p, d = batch
        f = [f] if isinstance(f, torch.Tensor) else [f[k] for k in sorted(f)]
        return f + [p[k] for k in sorted(p)] + [d]

    @staticmethod
    def _unflat(batch, flat):
        f, p, _ = batch
        if isinstance(f, torch.Tensor):
            return flat[0], {k: flat[1 + i] for i, k in enumerate(sorted(p))}, flat[-1]
        kf, kp = sorted(f), sorted(p)
        return ({k: flat[i] for i, k in enumerate(kf)}, {k: flat[len(kf) + i] for i, k in enumerate(kp)}, flat[-1])

    def _upload(self, slot, batch):
        host = self._flat(batch)
        if slot["bufs"] is None or any(b.shape != h.shape or b.stride() != h.stride() for b, h in zip(slot["bufs"], host)):
            # (re)allocation comes from the compute stream's allocator pool: the block may have just been freed by kernels
            # that are still queued on the compute stream, so the copy stream must not write it before they have run
            slot["bufs"] = [torch.empty_strided(h.shape, h.stride(), dtype=h.dtype, device=self.device) for h in host]
            self.copy_stream.wait_stream(torch.cuda.current_stream(self.device))
            for b in slot["bufs"]:
                b.record_stream(self.copy_stream)
                for lane in self.lanes:
                    b.record_stream(lane)
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(slot["free"])     # the kernels that read this slot have finished
            for b, h in zip(slot["bufs"], host):
                b.copy_(h, non_blocking=True)
            slot["ready"].record(self.copy_stream)
        # identity of the prefetched batch: a strong reference (id() alone can be reused by Python after the batch dies)
        slot["tag"], slot["batch"] = id(batch), batch

    def bytes_per_batch(self, batch):
        return sum(t.numel() * t.element_size() for t in self._flat(batch))

    @torch.no_grad()
    def run(self, batch, next_batch=None, tmp=(5.0, 5.0, 5.0, 1.0)):
        """Runs the hot path on `batch` (uploaded now unless a previous call prefetched it) and starts the upload of
        `next_batch` so that it overlaps this call's kernels.  Returns the reference's output dict (device tensors)."""
        cur = next((s for s in self.slots if s["batch"] is batch), None)
        if cur is None:
            cur = self.slots[self._next]
            self._next = (self._next + 1) % len(self.slots)
            self._upload(cur, batch)
        caller = torch.cuda.current_stream(self.device)
        compute = caller
        if self.lanes:
            # NOT ordered after the caller's stream: the caller's stream waits for lane i below, so such an edge would chain
            # lane i+1 behind lane i.  The batch comes from the copy stream, `tmp` from the host.
            compute = self.lanes[self._lane]
            self._lane = (self._lane + 1) % len(self.lanes)
        if next_batch is not None and not any(s["batch"] is next_batch for s in self.slots if s is not cur):
            others = [s for s in self.slots if s is not cur]
            nxt = next((s for s in others if s["batch"] is None), others[0])   # prefer a slot that holds no pending batch
            self._upload(nxt, next_batch)
        f, p, d = self._unflat(batch, cur["bufs"])
        with torch.cuda.stream(compute):
            compute.wait_event(cur["ready"])
            out = (self.net.forward if isinstance(f, torch.Tensor) else self.net.forward_features)(f, p, d, tmp)
            cur["free"].record(compute)
        cur["tag"] = cur["batch"] = None                   # consumed: the same host batch is uploaded again next time
        if self.lanes:
            # the caller consumes the outputs on ITS stream: order it after this lane (the other lane keeps running) and tell
            # the allocator that the tensors are in use there
            caller.wait_stream(compute)
            stack = [out]
            while stack:
                for v in stack.pop().values():
                    if isinstance(v, torch.Tensor):
                        v.record_stream(caller)
                    elif isinstance(v, dict):
                        stack.append(v)
        return out
