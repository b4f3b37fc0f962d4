"""Whole-network execution: a frozen quantized graph replayed as one CUDA graph per GPU.

``compile_model`` runs the frozen model once eagerly on ``IntActivation`` payloads (this builds and caches every
integer parameter: widened/permuted weights, bias integers, dyadic pairs), then captures a second run in a CUDA
graph.  Replays involve no Python, no allocation and no host synchronisation: ~55 fused kernels for ResNet-50.

Residual stream width: by default the post-ReLU residual stream is stored as uint16 (half the bytes of int32); every
kernel that narrows it raises a sticky device flag if a value exceeded 65535, in which case the batch is transparently
re-run with the int32 graph, so results are always exact (the reference does not clamp case-1 sums,
``utils/quantization_utils/quant_utils.py:456``).

Several engines: each CompiledModel owns a status word (its own library handle, ``ops.using_handle``), which its graphs
and eager runs reset, raise and copy, so engines replaying at the same time on other streams or threads neither hide nor
borrow each other's overflow flags.  Builds (warm-up and capture) run one at a time per process: torch captures on one
shared stream and synchronises the device when a capture begins.

Multi-GPU: the path shards over images with no data-path collective (SURVEY.md §8e); ``all_gather_logits`` is the one
NCCL exchange the benchmark config asks for.
"""
import threading

import torch

from . import ops, qtensor
from .eval_transform import MAX_SIDE, MIN_RESIZE, PackedImages, collate_images
from .modules import freeze_model
from .qtensor import IntActivation, Node


_BUILD_LOCK = threading.RLock()

IMAGENET_MEAN = (0.485, 0.456, 0.406)      # transforms.Normalize of the reference's loaders (quant_train.py:357-358,
IMAGENET_STD = (0.229, 0.224, 0.225)       # tvm_benchmark/test_resnet_accuracy_imagenet.py:82-83)


class CompiledModel:
    """input: int8 NHWC [N,H,W,3] (already quantised with the model's input scale), fp32 NCHW [N,3,H,W] (normalised, what the
    reference's loaders produce), or uint8 NHWC [N,H,W,3] raw pixels (ToTensor + Normalize(mean, std) + input quantisation are
    then one kernel at the head of the graph; needs ``model.quant_input``).

    With ``resize`` (the reference's evaluation transform, Resize(resize) -> CenterCrop(H, W) -> ToTensor -> Normalize): the input
    is a batch of up to N decoded RGB images of any sizes, a ``PackedImages`` or a list of HWC uint8 images, and the head kernel
    resizes, crops and quantises them on the device, bit-equal to torchvision on PIL.  The pixels go to a device arena (with a table
    of offsets and sizes) that the graphs read; a batch that does not fit grows it and recaptures the graphs (``recaptures``)."""

    def __init__(self, model, example, use_cuda_graph=True, residual_bits=16, mean=IMAGENET_MEAN, std=IMAGENET_STD, gather=False,
                 group=None, resize=None):
        if not example.is_cuda:
            raise RuntimeError("compile_model needs a CUDA example input: the frozen path has no CPU implementation")
        self.model = model
        self.device = example.device
        self.int_input = example.dtype == torch.int8
        self.u8_input = example.dtype == torch.uint8
        self.mean, self.std = tuple(mean), tuple(std)
        self.recaptures = 0
        if resize is not None and gather:
            raise NotImplementedError("resize with gather=True (sharded ragged batches) is not supported")
        if self.u8_input:
            if example.dim() != 4 or example.shape[-1] != 3:
                raise ValueError("uint8 input must be NHWC with 3 channels")
            act = getattr(model, "quant_input", None)
            if act is None or act.activation_bit != 8 or act.quant_mode != "symmetric":
                raise NotImplementedError("uint8 input needs an 8-bit symmetric `quant_input` QuantAct at the head of the model")
            self._q_in = torch.empty(example.numel(), dtype=torch.int8, device=example.device)
        self.resize = None if resize is None else int(resize)
        if self.resize is not None:
            if not self.u8_input:
                raise ValueError("resize needs a uint8 NHWC example: its H x W is the crop, its batch the number of image slots")
            self.slots, self.crop = example.shape[0], (example.shape[1], example.shape[2])
            if not MIN_RESIZE <= self.resize <= MAX_SIDE or self.resize < max(self.crop):
                raise ValueError("resize %d must lie in %d..%d and cover the crop %dx%d" % ((self.resize, MIN_RESIZE, MAX_SIDE) + self.crop))
            # the arena starts with room for 3 * resize^2 pixels per slot: a batch of ImageNet-sized images (500 x 375) fits
            self.arena = torch.zeros(self.slots * 3 * self.resize * self.resize * 3, dtype=torch.uint8, device=example.device)
            self.table = torch.zeros((self.slots, 2), dtype=torch.int64, device=example.device)   # hawq_image_desc rows; h = 0: absent
            self._n = self.slots
        self.static_in = example.clone() if self.resize is None else None
        self.use_graph = use_cuda_graph
        self.flag = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.gather, self.group = bool(gather), group
        if self.gather:
            import torch.distributed as dist
            self.all_flags = torch.zeros(dist.get_world_size(group), dtype=torch.int32, device=self.device)
        self.graphs = {}
        self.outs = {}
        self.gathered = {}
        self.launches = {}
        self.residual_bits = residual_bits
        self.input_scale = None
        self.fallbacks = 0
        self._handle = ops.acquire_handle(self.device.index)     # this engine's status word, baked into every graph it captures
        with torch.no_grad():
            self._build(residual_bits)

    def __del__(self):
        h = self.__dict__.pop("_handle", None)
        if h is not None:
            self.graphs.clear()                 # the graphs that write this handle's word go first
            ops.release_handle(self.device.index, h)

    # -- one eager forward on the current stream
    def _forward(self, bits, fast=True):
        with qtensor.engine_mode(residual_bits=bits, fast_kernels=fast, checked=True):
            return self._forward_checked()

    def _forward_checked(self):
        x = self.static_in
        if self.resize is not None:
            act = self.model.quant_input
            ops.resize_crop_quantize_u8(self.arena, self.table, self.resize, self.crop, self.mean, self.std, float(qtensor._frozen_scale(act)),
                                        qtensor._act_clamp(act), self._q_in)
            x = IntActivation(Node("int", (self.slots, 3) + self.crop, data=self._q_in, bits=8, signed=True), self.device)
        elif self.u8_input:
            act = self.model.quant_input
            ops.quantize_input_u8(x, self.mean, self.std, float(qtensor._frozen_scale(act)), qtensor._act_clamp(act), self._q_in)
            n, h, w, c = x.shape
            x = IntActivation(Node("int", (n, c, h, w), data=self._q_in, bits=8, signed=True), self.device)
        elif self.int_input:
            n, h, w, c = x.shape
            x = IntActivation(Node("int", (n, c, h, w), data=x.view(-1), bits=8, signed=True), self.device)
        return self.model(x)

    def _build(self, bits, key=None):
        with _BUILD_LOCK, ops.using_handle(self.device.index, self._handle):
            self._build_locked(bits, key)

    def _build_locked(self, bits, key):
        key = bits if key is None else key
        fast = key != "safe"                    # "safe": no ratio promises -> saturating generic kernels
        idx = self.device.index
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            before = ops.thread_launch_count()
            out = self._forward(bits, fast)            # warm-up: builds all parameter caches
            self.launches[key] = ops.thread_launch_count() - before
            out = self._forward(bits, fast)
            if self.gather:
                self.gathered[key] = all_gather_logits(out, self.group)   # also initialises the NCCL communicator before capture
        # keep every module's plan (device-resident weights / per-channel parameters) alive for as long as graphs captured
        # here may replay, even if the modules drop or rebuild theirs (unfix(), load_state_dict)
        self._plans = getattr(self, "_plans", [])
        self._plans.append([m.__dict__["_hawq_cache"] for m in self.model.modules() if "_hawq_cache" in m.__dict__])
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        self.bits_of = getattr(self, 'bits_of', {})
        self.bits_of[key] = bits
        if not self.use_graph:
            self.outs[key] = out
            return
        g = torch.cuda.CUDAGraph()
        # thread_local: other threads may allocate, synchronise and launch (eager runs, replays) while this capture is underway
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            ops.reset_status(idx)
            out = self._forward(bits, fast)
            ops.copy_status(idx, self.flag)
            if self.gather:                     # the path's one collective rides inside the graph: no extra launch / host work per step
                self.gathered[key] = all_gather_logits(out, self.group)
                self._gather_flags()
        self.graphs[key] = g
        self.outs[key] = out

    def _run(self, key):
        if self.use_graph:
            self.graphs[key].replay()
        else:
            with ops.using_handle(self.device.index, self._handle):
                ops.reset_status(self.device.index)
                self.outs[key] = self._forward(self.bits_of[key], key != "safe")
                ops.copy_status(self.device.index, self.flag)
            if self.gather:
                self.gathered[key] = all_gather_logits(self.outs[key], self.group)
                self._gather_flags()
        return self.outs[key]

    def _gather_flags(self):
        """Sharded runs: every rank sees every rank's status word, so all ranks take the same (exact) fallback together."""
        import torch.distributed as dist
        dist.all_gather_into_tensor(self.all_flags, self.flag, group=self.group)

    def _flags(self, host_flags=None):
        if self.gather:
            v = 0
            for f in (self.all_flags.tolist() if host_flags is None else host_flags):
                v |= int(f)
            return v
        return int(self.flag.item()) if host_flags is None else int(host_flags[0])

    def _result(self, key):
        return self.gathered[key] if self.gather else self.outs[key]

    def _grow(self, nbytes):
        """A bigger arena for a batch of ``nbytes`` pixel bytes: every graph is recaptured over it."""
        torch.cuda.synchronize(self.device)                  # no replay still reads the old arena
        self.arena = torch.zeros(nbytes * 5 // 4, dtype=torch.uint8, device=self.device)
        keys = list(self.outs)
        self.graphs.clear()
        with torch.no_grad():
            for key in keys:
                self._build(self.bits_of[key], key=key)
        self.recaptures += 1

    def _packed(self, images):
        p = images if isinstance(images, PackedImages) else collate_images(list(images))
        if len(p) > self.slots:
            raise ValueError("%d images for %d slots" % (len(p), self.slots))
        if p.pixels.numel() > self.arena.numel():
            self._grow(p.pixels.numel())
        return p

    def _stage(self, images):
        p = self._packed(images)
        self.arena[:p.pixels.numel()].copy_(p.pixels, non_blocking=True)
        self.table.copy_(p.table(self.slots), non_blocking=True)
        self._n = len(p)

    def run_async(self, x=None):
        """Enqueue one forward (no host sync, no overflow check); returns the static logits tensor (with ``gather`` the logits
        of the whole sharded batch, gathered from every rank inside the same CUDA graph; with ``resize`` all N rows, the rows past
        the batch's images belonging to absent slots)."""
        if x is not None and self.resize is not None:
            self._stage(x)
        elif x is not None:
            self.static_in.copy_(x, non_blocking=True)
        out = self._run(self.residual_bits)
        return self.gathered[self.residual_bits] if self.gather else out

    def __call__(self, x=None):
        """Exact forward: replays the fast graph, checks the overflow flag, falls back to int32 residuals if needed.  With ``resize``
        the logits of the batch's n images, [n, classes]."""
        out = self._call(x)
        return out if self.resize is None else out[:self._n]

    def _call(self, x):
        out = self.run_async(x)
        self._last_key = self.residual_bits
        flags = self._flags()
        if flags & 2:
            raise RuntimeError("hawq_b200: HAWQ_FLAG_BAD_RATIO raised (a dyadic ratio > 1 reached the fast kernel): results invalid")
        if flags & 4:                          # a ratio > 1 term left int32 on the fast path: saturating generic kernels
            self.fallbacks += 1
            with torch.no_grad():
                if "safe" not in self.outs:
                    self._build(32, key="safe")
                self._run("safe")
            self._last_key = "safe"
            return self._result("safe")
        if self.residual_bits == 16 and flags & 1:
            self.fallbacks += 1
            if 32 not in self.outs:
                with torch.no_grad():
                    self._build(32)
            self._run(32)
            self._last_key = 32
            return self._result(32)
        return out

    def run_pipelined(self, host_batches, post=None):
        """Exact forward over an iterable of pinned host batches with copy/compute overlap: the H2D copy of batch i+1 runs on a
        copy stream while batch i computes; logits and the status flags come back through pinned buffers and are checked one
        step later (a raised overflow flag re-runs that batch through ``__call__``, i.e. the exact int32 / saturating graphs).
        ``post`` is applied to the device logits before they are read back.  With ``gather`` the logits of the whole sharded batch
        stay on the device (``self.gathered``) and the host reads this rank's shard.  With ``resize`` a batch is a ``PackedImages``
        (pinned, for a copy that overlaps) or a list of images, and its rows are those of its images; the staging buffers grow
        with the arena.
        Yields the host logits tensor of every batch, in order (valid until the second next iteration)."""
        dev = self.device
        main = torch.cuda.current_stream(dev)
        if not hasattr(self, "_pipe"):
            cs = torch.cuda.Stream(device=dev)
            out = self.outs[self.residual_bits]
            if post is not None:
                out = post(out)
            # three host logits buffers: batch i's is yielded during iteration i + 1 and must survive iteration i + 2, which
            # already enqueues the read-back of batch i + 2
            src = self.static_in if self.resize is None else self.arena
            self._pipe = dict(copy=cs, stage=[torch.empty_like(src) for _ in range(2)],
                              table=[torch.empty_like(self.table) for _ in range(2)] if self.resize is not None else None,
                              out=[torch.empty(out.shape, dtype=out.dtype).pin_memory() for _ in range(3)],
                              flag=[torch.zeros(self.all_flags.numel() if self.gather else 1, dtype=torch.int32).pin_memory() for _ in range(2)],
                              h2d=[torch.cuda.Event() for _ in range(2)], free=[torch.cuda.Event() for _ in range(2)],
                              done=[torch.cuda.Event() for _ in range(2)])
        P = self._pipe
        prev = None

        def finish(slot, oslot, xb, n):
            P["done"][slot].synchronize()
            if self._flags(P["flag"][slot].tolist()) & 7:
                self(xb)                            # rare: exact fallback path, synchronous (sharded runs: every rank takes it together)
                out = self.outs[self._last_key]
                return (post(out) if post is not None else out).to("cpu")[:n]
            return P["out"][oslot][:n]

        for i, xb in enumerate(host_batches):
            slot, oslot = i & 1, i % 3
            n = None
            if self.resize is not None:
                xb = self._packed(xb)
                n, nb = len(xb), xb.pixels.numel()
                if nb > P["stage"][0].numel():
                    torch.cuda.synchronize(dev)     # neither stage buffer is still being copied
                    P["stage"] = [torch.empty_like(self.arena) for _ in range(2)]
            with torch.cuda.stream(P["copy"]):
                P["copy"].wait_event(P["free"][slot])
                if self.resize is None:
                    P["stage"][slot].copy_(xb, non_blocking=True)
                else:
                    P["stage"][slot][:nb].copy_(xb.pixels, non_blocking=True)
                    P["table"][slot].copy_(xb.table(self.slots), non_blocking=True)
                P["h2d"][slot].record(P["copy"])
            main.wait_event(P["h2d"][slot])
            if self.resize is None:
                self.static_in.copy_(P["stage"][slot], non_blocking=True)
            else:
                self.arena[:nb].copy_(P["stage"][slot][:nb], non_blocking=True)
                self.table.copy_(P["table"][slot], non_blocking=True)
                self._n = n
            P["free"][slot].record(main)
            out = self._run(self.residual_bits)
            if post is not None:
                out = post(out)
            P["out"][oslot].copy_(out, non_blocking=True)
            P["flag"][slot].copy_(self.all_flags if self.gather else self.flag, non_blocking=True)
            P["done"][slot].record(main)
            if prev is not None:
                yield finish(*prev)
            prev = (slot, oslot, xb, n)
        if prev is not None:
            yield finish(*prev)

    @property
    def gpu_launches(self):
        return self.launches.get(self.residual_bits, 0)

    def save(self, path):
        """Write this engine as one plan file (engine_file.py): its fast, int32 and safe forwards, recorded launch by launch, with
        the weights and tables they read.  ``hawq_b200.load_engine`` or the C runtime (include/hawq_b200.h) runs it without the model.
        Builds the fallback graphs not built yet.  Not for ``resize`` or ``gather`` engines (NotImplementedError).  Returns the
        file's size in bytes."""
        from . import engine_file
        return engine_file.save(self, path)


def compile_model(model, example, use_cuda_graph=True, residual_bits=16, mean=IMAGENET_MEAN, std=IMAGENET_STD, gather=False, group=None,
                  resize=None):
    """Freeze ``model`` (a QResNet or any graph built from hawq_b200.modules) and compile it for ``example``'s shape and dtype
    (int8 NHWC, fp32 NCHW or uint8 NHWC; ``mean`` / ``std`` only matter for uint8 pixels).  ``gather``: the batch is sharded over the
    ranks of ``group`` (torch.distributed, NCCL) and every forward all-gathers the logits inside the CUDA graph.  ``resize``: with a
    uint8 NHWC example [N, H, W, 3], the engine takes up to N decoded images of any sizes and applies Resize(resize) + CenterCrop(H, W)
    on the device (see CompiledModel)."""
    freeze_model(model)
    model.eval()
    return CompiledModel(model, example, use_cuda_graph=use_cuda_graph, residual_bits=residual_bits, mean=mean, std=std, gather=gather,
                         group=group, resize=resize)


def all_gather_logits(local_logits, group=None):
    """The single collective of the sharded path: gather [B/G, classes] fp32 logits from every rank (NCCL)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    out = torch.empty((world * local_logits.shape[0], local_logits.shape[1]), dtype=local_logits.dtype,
                      device=local_logits.device)
    dist.all_gather_into_tensor(out, local_logits.contiguous(), group=group)
    return out


def shard_range(total, rank, world):
    """Images [lo, hi) of a batch of ``total`` handled by ``rank`` (contiguous, remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
