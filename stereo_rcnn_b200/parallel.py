"""Multi-GPU plumbing of the hot path: independent stereo pairs shard over ranks (one process per
GPU, torch.distributed), and the only exchange is ONE all-gather of the fixed-size per-image
detection record (SURVEY 8e).  No data-path collective exists anywhere else: BN is frozen, every
stage is per-image or per-RoI.
"""
import torch

REC_ROIS = 300
REC_COLS = 2 + 8 + 8 + 10 + 5        # cls scores, boxes L/R (per class), dim/orientation, keypoints


def shard_pairs(n_pairs, rank, world):
    """contiguous split of a batch of stereo pairs; returns the [begin, end) range of this rank"""
    base, rem = divmod(n_pairs, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def detection_record(cls_prob, pred_boxes_left, pred_boxes_right, dim_orien, pred_kpts):
    """[R, 33] fp32 record of one image (what test_net.py:233-330 consumes downstream)"""
    return torch.cat((cls_prob, pred_boxes_left, pred_boxes_right, dim_orien, pred_kpts), 1)


def gather_records(rec, world, dist=None, out=None):
    """all-gather of one record per rank -> [world, R, C] (identity for world == 1)"""
    if world == 1:
        return rec.unsqueeze(0)
    if out is None:
        out = torch.empty((world,) + tuple(rec.shape), dtype=rec.dtype, device=rec.device)
    # dim-0 concatenation layout (accepted by both NCCL and gloo)
    dist.all_gather_into_tensor(out.view((-1,) + tuple(rec.shape[1:])), rec.contiguous())
    return out


def max_over_ranks(value_ms, device, world, dist=None):
    """device-timed duration reduced with MAX over ranks (the bench contract)"""
    if world == 1:
        return float(value_ms)
    t = torch.tensor([float(value_ms)], device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


class RecordGather(object):
    """The exchange step: `gather(slot, rec [R, C]) -> [world, R, C]`, one call per step and in-flight slot.

    mode "nccl" (default): one `all_gather_into_tensor` per step on a process group PRIVATE to the slot (a communicator
        used from several streams would serialise the slots on ProcessGroupNCCL's internal stream -- round 1's 0.942).
    mode "peer": the ranks store their record straight into each other's mailboxes over NVLink and release a
        sequence flag (csrc/peer.cu; CUDA IPC handles travel once through torch.distributed); optionally pipelined
        (lag 1).  No NCCL kernel on the data path.  Verified bit-exact on 2 / 4 / 8 GPUs, but measured 2-3 % behind the
        per-slot NCCL communicators on the bench (N = 2: 596 vs 613 pairs/s, N = 8: 2321 vs 2388), so it is opt-in.
        When R * C is not a multiple of 4, the result is a row-strided view of a [world, R * C rounded up to 4] buffer.
    On CPU tensors (gloo host tests) the collective is always torch.distributed's.
    world == 1: identity.  `describe()` says which path is live; a peer set-up failure is reported there, not hidden.
    """

    def __init__(self, world, rank, device, dist=None, n_slots=1, mode=None, rec_shape=(REC_ROIS, REC_COLS),
                 timeout_s=20.0, lag=0):
        """lag = 1 (peer mode only): pipelined exchange -- a call puts this step's record and returns the gathered
        records of the slot's PREVIOUS step, so that no rank ever waits for a slower peer's current step; `drain(slot)`
        collects the last step.  lag = 0: the gathered records of this very step (what a collective gives)."""
        import os
        self.world, self.rank, self.dist, self.n_slots = world, rank, dist, n_slots
        self.device = torch.device(device)
        self.rec_shape = tuple(rec_shape)
        self.rec_floats = (int(rec_shape[0] * rec_shape[1]) + 3) // 4 * 4
        self.timeout_s = timeout_s
        self.lag = int(lag)
        mode = mode or os.environ.get("SB_GATHER", "nccl")
        self.mode = "none" if world == 1 else ("nccl" if self.device.type != "cuda" else mode)
        self.note = ""
        if self.mode == "peer":
            try:
                self._setup_peer()
            except Exception as e:      # reported in describe() and in the bench line
                self.note = "peer set-up failed (%s: %s), using nccl" % (type(e).__name__, e)
                self.mode = "nccl"
            # every rank must take the same path
            ok = torch.tensor([1 if self.mode == "peer" else 0], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
            if int(ok[0]) == 0 and self.mode == "peer":
                self.mode, self.note = "nccl", "a peer rank could not map the mailboxes, using nccl"
        if self.mode == "peer":
            # the wait copies every rank's whole padded record (rec_floats floats, a float4 multiple) at a rec_floats
            # stride, so a slot's output is a [world, rec_floats] buffer seen as [world, R, C]
            n = self.rec_shape[0] * self.rec_shape[1]
            self._gathered = [torch.empty(world, self.rec_floats, dtype=torch.float32, device=self.device)
                              for _ in range(n_slots)]
            self.out = [g[:, :n].view((world,) + self.rec_shape) for g in self._gathered]
        else:
            self.lag = 0
            self.out = [torch.empty((world,) + self.rec_shape, dtype=torch.float32, device=self.device)
                        for _ in range(n_slots)] if world > 1 else None
        if self.mode == "nccl":
            self.groups = [dist.new_group() if self.device.type == "cuda" else None for _ in range(n_slots)]

    # ---- peer path ----
    def _setup_peer(self):
        import ctypes
        from . import lib
        L = lib.load()
        nb = L.sb_peer_mailbox_bytes(self.n_slots, self.world, self.rec_floats)
        if nb == 0:
            raise ValueError("unsupported mailbox geometry")
        own = ctypes.c_void_p()
        lib.check(L.sb_peer_alloc(nb, ctypes.byref(own)), "sb_peer_alloc")
        h = (ctypes.c_ubyte * 64)()
        lib.check(L.sb_ipc_export(own, h), "sb_ipc_export")
        mine = torch.tensor(list(h), dtype=torch.uint8, device=self.device)
        allh = torch.empty(self.world, 64, dtype=torch.uint8, device=self.device)
        self.dist.all_gather_into_tensor(allh.view(-1), mine)
        allh = allh.cpu()
        self._boxes = (ctypes.c_void_p * self.world)()
        for r in range(self.world):
            if r == self.rank:
                self._boxes[r] = own.value
            else:
                hb = (ctypes.c_ubyte * 64)(*allh[r].tolist())
                p = ctypes.c_void_p()
                lib.check(L.sb_ipc_import(hb, ctypes.byref(p)), "sb_ipc_import(rank %d)" % r)
                self._boxes[r] = p.value
        self._own = own
        self._err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._staged = [torch.zeros(self.rec_floats, dtype=torch.float32, device=self.device)
                        for _ in range(self.n_slots)]
        self.dist.barrier()

    def check(self):
        """host-side: raise if a wait timed out (reads one device int; call outside timed regions)"""
        if self.mode == "peer":
            e = int(self._err[0])
            if e:
                raise RuntimeError("record gather: rank %d never delivered" % (e - 1))

    def __call__(self, slot, rec):
        if self.world == 1:
            return rec.unsqueeze(0)
        out = self.out[slot]
        if self.mode == "peer":
            from . import lib
            L = lib.load()
            n = rec.numel()
            src = rec
            if n != self.rec_floats or not rec.is_contiguous() or rec.data_ptr() % 16:
                src = self._staged[slot]
                src[:n].copy_(rec.reshape(-1))
            st = lib.stream_ptr()
            lib.check(L.sb_peer_put_record(lib.ptr(src), self._boxes, self.n_slots, self.world, self.rec_floats,
                                           self.rank, slot, st), "sb_peer_put_record")
            lib.check(L.sb_peer_wait_records(self._own, self.n_slots, self.world, self.rec_floats, slot, self.lag,
                                             lib.ptr(self._gathered[slot]), lib.ptr(self._err), float(self.timeout_s),
                                             st),
                      "sb_peer_wait_records")
            return out
        self.dist.all_gather_into_tensor(out.view((-1,) + self.rec_shape[1:]), rec.contiguous(),
                                         group=self.groups[slot])
        return out

    def drain(self, slot):
        """lag = 1: collect the records of the slot's LAST step (no new put) -> [world, R, C]; otherwise a no-op"""
        if self.world == 1 or self.mode != "peer" or self.lag == 0:
            return None if self.out is None else self.out[slot]
        from . import lib
        L = lib.load()
        lib.check(L.sb_peer_wait_records(self._own, self.n_slots, self.world, self.rec_floats, slot, 0,
                                         lib.ptr(self._gathered[slot]), lib.ptr(self._err), float(self.timeout_s),
                                         lib.stream_ptr()),
                  "sb_peer_wait_records")
        return self.out[slot]

    def describe(self):
        if self.world == 1:
            return "none (1 GPU)"
        d = {"peer": "own kernels over NVLink peer memory (CUDA IPC mailboxes, posted 128-bit stores + release flags%s)"
                     % (", pipelined: a step collects the previous step's records" if self.lag else ""),
             "nccl": "ncclAllGather (torch.distributed.all_gather_into_tensor), one communicator per in-flight slot"}[self.mode]
        return d + ("; " + self.note if self.note else "")


class GradientBuckets(object):
    """Data-parallel gradient exchange of a training step (SURVEY 8e / config 4: the batch shards over the GPUs,
    gradients are averaged; the reference uses nn.DataParallel inside one process, trainval_net.py:186-187).

    The gradient tensors ARE views into a few flat fp32 buckets (`grads[i]`, same shapes as the parameters): kernels
    write gradients in place, `all_reduce()` issues one NCCL all-reduce per bucket -- no flatten / unflatten copies --
    and divides by the world size.  Buckets are sized for launch latency, not link count (NVSwitch: every GPU has full
    bandwidth to every peer): 64 MB default, ResNet-101's ~190 MB of fp32 gradients travel in 3 collectives.
    `clip()` is net_utils.clip_gradient over the same views (one global norm on the device, no per-parameter sync).
    world == 1 or dist None: all_reduce() is the identity."""

    def __init__(self, shapes, device, world=1, dist=None, bucket_bytes=64 << 20):
        self.world, self.dist, self.device = int(world), dist, torch.device(device)
        self.buckets, self.grads = [], []
        cap = max(int(bucket_bytes) // 4, 1)
        plan, cur, cur_n = [], [], 0
        for shp in shapes:
            n = 1
            for d in shp:
                n *= int(d)
            n_pad = (n + 3) // 4 * 4                     # keep every view 16-byte aligned inside its bucket
            if cur and cur_n + n_pad > cap:
                plan.append((cur, cur_n))
                cur, cur_n = [], 0
            cur.append((tuple(int(d) for d in shp), n, cur_n))
            cur_n += n_pad
        if cur:
            plan.append((cur, cur_n))
        for entries, total in plan:
            flat = torch.zeros(total, dtype=torch.float32, device=self.device)
            self.buckets.append(flat)
            for shp, n, off in entries:
                self.grads.append(flat[off:off + n].view(shp))

    def zero_(self):
        for b in self.buckets:
            b.zero_()

    def all_reduce(self):
        """sum over ranks / world, in place (stream-ordered on the current stream for NCCL)"""
        if self.world == 1 or self.dist is None:
            return self
        for b in self.buckets:
            self.dist.all_reduce(b, op=self.dist.ReduceOp.SUM)
            b.div_(self.world)
        return self

    def clip(self, clip_norm):
        """net_utils.clip_gradient (net_utils.py:37-49) on the device -> [total norm, applied factor]"""
        if self.device.type != "cuda":                   # host tests: same arithmetic in torch
            total = torch.sqrt(sum((g.double() ** 2).sum() for g in self.grads)).float()
            f = float(clip_norm) / max(float(total), float(clip_norm))
            for b in self.buckets:
                b.mul_(f)
            return torch.tensor([float(total), f])
        from . import train
        return train.clip_gradient(self.grads, clip_norm)

    def describe(self):
        return "%d gradient tensors in %d flat buckets (%s MB), %s" % (
            len(self.grads), len(self.buckets), "+".join("%.1f" % (b.numel() * 4 / 2 ** 20) for b in self.buckets),
            "ncclAllReduce per bucket, averaged" if self.world > 1 and self.dist is not None else "single rank")


def average_losses(losses, world, dist=None):
    """mean of the per-rank loss vector (what trainval_net.py logs after DataParallel's `.mean()`, :214-219)"""
    if world == 1 or dist is None:
        return losses
    out = losses.clone()
    dist.all_reduce(out, op=dist.ReduceOp.SUM)
    return out / world
