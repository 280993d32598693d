"""Device policy and host<->device frame streaming shared by the node classes."""
import math
import os
import threading

import torch

from .dist import shard_range


def _comfy_mm():
    try:
        import comfy.model_management as mm  # provided by the ComfyUI host process
        return mm
    except Exception:
        return None


def compute_device(hint=None):
    """The CUDA device the kernels run on.  Mirrors comfy.model_management.get_torch_device() (nodes.py:42);
    outside ComfyUI: the tensor's own CUDA device, else the current CUDA device.  Never a CPU."""
    if isinstance(hint, torch.Tensor) and hint.device.type == "cuda":
        return hint.device
    mm = _comfy_mm()
    if mm is not None:
        dev = torch.device(mm.get_torch_device())
        if dev.type == "cuda":
            return dev
    if not torch.cuda.is_available():
        raise RuntimeError("vrgdg_b200: no CUDA device is available; these nodes are sm_90a kernels and have no CPU path")
    return torch.device("cuda", torch.cuda.current_device())


def cuda_device(d):
    """torch.device of a CUDA device with its index filled in ("cuda" = the current device); anything else is a ValueError."""
    d = torch.device(d)
    if d.type != "cuda":
        raise ValueError("vrgdg_b200: %s is not a CUDA device; these kernels have no CPU path" % d)
    return d if d.index is not None else torch.device("cuda", torch.cuda.current_device())


def devices_from_env():
    """The CUDA devices VRGDG_DEVICES names for sharding host IMAGE batches, or None when it is unset or empty (the one compute
    device).  "all" = every visible device of compute capability 9.0; otherwise a comma-separated list of device indices, each
    visible, of compute capability 9.0 and listed once (a repeated index is most likely a typo for another card)."""
    raw = os.environ.get("VRGDG_DEVICES", "").strip()
    if not raw:
        return None
    n = torch.cuda.device_count()
    if raw.lower() == "all":
        idx = [i for i in range(n) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
        if not idx:
            raise ValueError("VRGDG_DEVICES=all: none of the %d visible CUDA devices has compute capability 9.0" % n)
        return [torch.device("cuda", i) for i in idx]
    idx = []
    for tok in raw.split(","):
        tok = tok.strip()
        try:
            i = int(tok)
        except ValueError:
            raise ValueError("VRGDG_DEVICES=%s: %r is not a device index (use 'all' or a list such as 0,1)" % (raw, tok)) from None
        if not 0 <= i < n:
            raise ValueError("VRGDG_DEVICES=%s: there is no device cuda:%d (%d visible)" % (raw, i, n))
        if i in idx:
            raise ValueError("VRGDG_DEVICES=%s: device cuda:%d is listed twice" % (raw, i))
        cap = tuple(torch.cuda.get_device_capability(i))
        if cap != (9, 0):
            raise ValueError("VRGDG_DEVICES=%s: device cuda:%d (%s) has compute capability %d.%d; the kernels are sm_90a code for 9.0 only"
                             % (raw, i, torch.cuda.get_device_name(i), cap[0], cap[1]))
        idx.append(i)
    return [torch.device("cuda", i) for i in idx]


# noise sources of the grain: "vrgdg" = this package's counter-based generator, "torch_cuda" = torch's CUDA randn stream
NOISE_STREAMS = ("vrgdg", "torch_cuda")


def grain_noise_from_env():
    """FastFilmGrain's noise source, VRGDG_GRAIN_NOISE: unset, empty or "vrgdg" = this package's generator (the default);
    "torch_cuda" = the draws the reference makes from the compute device's global CUDA generator.  Read at call time."""
    raw = os.environ.get("VRGDG_GRAIN_NOISE", "").strip()
    if raw in ("",) + NOISE_STREAMS:
        return raw or NOISE_STREAMS[0]
    raise ValueError("VRGDG_GRAIN_NOISE=%s: use one of %s" % (raw, " or ".join(NOISE_STREAMS)))


def result_device(images, numpy_path=False):
    """Where a node returns its IMAGE.  Inside ComfyUI: exactly what the reference does
    (intermediate_device() nodes.py:65,123,177; CPU for the numpy paths :209).  Outside: the input's device."""
    mm = _comfy_mm()
    if mm is not None:
        return torch.device("cpu") if numpy_path else torch.device(mm.intermediate_device())
    return images.device


_SIDE_STREAMS = {}


def _pin_result(src, nbytes):
    """Host results are allocated pinned when the source is pinned, or when they are small enough (VRGDG_PIN_RESULT_BYTES, default
    2 GiB): the download then runs at PCIe speed instead of through the driver's pageable bounce buffer, and the next node's upload of
    that tensor does too.  torch caches freed pinned blocks, so repeated runs of a workflow do not pay cudaHostAlloc again."""
    import os
    if src.is_pinned():
        return True
    try:
        limit = int(os.environ.get("VRGDG_PIN_RESULT_BYTES", str(2 << 30)))
    except ValueError:
        limit = 2 << 30
    return 0 < nbytes <= limit


def _env_bytes(name, default):
    import os
    try:
        return int(os.environ.get(name, str(default)))
    except ValueError:
        return default


def upload(t, dev):
    """One host tensor to the device.  Large pageable tensors (a 4K reference frame is 99.5 MB) go through a pinned staging buffer
    filled by torch's multi-threaded host copy instead of the driver's single-threaded bounce copy; torch's host allocator keeps the
    staging block alive until the copy has finished and caches it for the next call.  CUDA tensors and small ones: plain .to()."""
    if t.device.type != "cpu" or t.is_pinned() or t.numel() * t.element_size() < (8 << 20) or _env_bytes("VRGDG_STAGE_PAGEABLE", 1) <= 0:
        return t.to(dev)
    try:
        stage = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    except RuntimeError:
        return t.to(dev)
    stage.copy_(t)
    return stage.to(dev, non_blocking=True)


def pipeline_chunk(chunk, frame_bytes, cap=None):
    """Frames per pipeline chunk for host sources: the caller's chunk, cut down to VRGDG_STREAM_CHUNK_BYTES (default 256 MiB; 0 = no
    cap), never below one frame."""
    cap = _env_bytes("VRGDG_STREAM_CHUNK_BYTES", 256 << 20) if cap is None else int(cap)
    if cap <= 0:
        return max(1, int(chunk))
    return max(1, min(int(chunk), cap // max(1, int(frame_bytes))))


_SIDE_STREAMS_LOCK = threading.Lock()


def _side_streams(dev, lane=0):
    """(upload, download) streams of a device, created once (stream creation is not free and ComfyUI calls nodes repeatedly).
    `lane` k > 0 is the k-th extra pair of the device, for a sharded call that runs several workers on one card."""
    key = (dev.type, dev.index, lane)
    with _SIDE_STREAMS_LOCK:                    # the workers of stream_frames_sharded ask from their own threads
        hit = _SIDE_STREAMS.get(key)
        if hit is None:
            hit = _SIDE_STREAMS[key] = (torch.cuda.Stream(dev), torch.cuda.Stream(dev))
    return hit


def bind_to_gpu_numa(device_index):
    """Pin this process to the CPUs NVML reports as local to GPU `device_index` (its NUMA node).  Call BEFORE allocating /
    first-touching pinned host buffers: a rank that stages frames through the other socket's memory pays the inter-socket
    link on every PCIe transfer.  Returns the CPU list, or None when NVML / sched_setaffinity are unavailable."""
    import os
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(int(device_index))
        words = (os.cpu_count() + 63) // 64
        mask = pynvml.nvmlDeviceGetCpuAffinity(h, words)
        cpus = [w * 64 + b for w, m in enumerate(mask) for b in range(64) if (int(m) >> b) & 1]
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return allowed
    except Exception:
        return None


def _result_shape(src, out_frame_shape):
    """Shape of the streamed result: the source's, or [B, *out_frame_shape] for a fn whose frames change shape."""
    return tuple(src.shape) if out_frame_shape is None else (int(src.shape[0]),) + tuple(int(d) for d in out_frame_shape)


def _check_out(out, shape, dtype, out_device):
    if tuple(out.shape) != tuple(shape) or out.dtype != dtype or out.device != out_device:
        raise ValueError("vrgdg_b200: `out` must be a %s tensor of the result's shape %s on %s" % (dtype, list(shape), out_device))


def stream_frames(src, fn, chunk, out_device, device=None, out=None, depth=2, lane=0, out_frame_shape=None):
    """Apply fn(cuda_frames, first_frame_index) -> cuda_frames over src [B,...] in chunks of `chunk` frames (0 / None = all).

    CUDA input: chunked as well (the reference bounds device memory with its batch_size widget the same way, nodes.py:49-62);
    one call when the chunk covers the batch.  CPU input: a three-stream pipeline - chunk k+1.. are uploaded into `depth`+1
    reusable staging buffers while chunk k computes and earlier results download; only the last download is waited for.
    Pinned source / result tensors make the copies truly asynchronous (the result is pinned when the source is).  `out`:
    optional preallocated result on out_device (reused across calls so that pinning cost is paid once).  `lane`: which pair of
    the device's upload / download streams carries the copies (stream_frames_sharded gives each worker on a card its own).
    `out_frame_shape`: the shape of one result frame when fn changes it (a resample); fn then returns [n, *out_frame_shape] in the
    source dtype, pipeline chunks are sized on the larger of an input and a result frame, and fn is called for a host chunk only once
    the result of the chunk `depth`+1 before it has downloaded, so results larger than their inputs cannot pile up on the device
    while the download falls behind.  None: result frames have the source frames' shape."""
    B = int(src.shape[0])
    out_device = torch.device(out_device)
    chunk = B if chunk is None or int(chunk) <= 0 else min(int(chunk), max(B, 1))
    out_shape = _result_shape(src, out_frame_shape)
    out_bytes = math.prod(out_shape) * src.element_size()
    if src.device.type == "cuda":
        if chunk >= B:
            res = fn(src, 0)
            return res if res.device == out_device else res.to(out_device)
        to_host = out_device.type == "cpu"
        res = torch.empty(out_shape, dtype=src.dtype, device=out_device, pin_memory=to_host and _pin_result(src, out_bytes))
        for i in range(0, B, chunk):
            res[i:i + chunk].copy_(fn(src[i:i + chunk], i), non_blocking=to_host)
        if to_host:
            torch.cuda.current_stream(src.device).synchronize()
        return res
    dev = device if device is not None else compute_device()
    if B == 0:
        if out_frame_shape is not None:
            return torch.empty(out_shape, dtype=src.dtype, device=out_device)
        return torch.empty_like(src, device=out_device)
    src = src.contiguous()
    to_cpu = out_device.type == "cpu"
    # Host frames move in pipeline chunks of at most VRGDG_STREAM_CHUNK_BYTES (default 256 MiB, at least one frame): a chunk as large
    # as the batch would serialise upload, kernels and download.  Every caller's fn is independent of how the batch is cut (noise is
    # keyed by the absolute frame index, statistics are per frame, temporal neighbours are fetched by index).  The cap holds for the
    # larger of a source and a result frame, so that an upscale's result chunk stays within it too.
    chunk = pipeline_chunk(chunk, max(src[0].numel() * src.element_size(), out_bytes // B))
    # A pageable source is staged through two pinned buffers by a multi-threaded host copy (torch's CPU copy_), so the DMA engine
    # reads pinned memory at PCIe speed while the next chunk is staged; the driver's own pageable path is a single-threaded bounce copy.
    stage = None
    if not src.is_pinned() and _env_bytes("VRGDG_STAGE_PAGEABLE", 1) > 0:
        try:
            stage = [torch.empty((chunk,) + tuple(src.shape[1:]), dtype=src.dtype, pin_memory=True) for _ in range(2)]
        except RuntimeError:
            stage = None                         # no pinned memory to spare: the driver's pageable path still works
    stage_free = [None, None]
    with torch.cuda.device(dev):
        compute = torch.cuda.current_stream(dev)
        up, down = _side_streams(dev, lane)
        if out is None:
            out = torch.empty(out_shape, dtype=src.dtype, pin_memory=_pin_result(src, out_bytes)) if to_cpu \
                else torch.empty(out_shape, dtype=src.dtype, device=out_device)
        else:
            _check_out(out, out_shape, src.dtype, out_device)
        n_chunks = (B + chunk - 1) // chunk
        slots = [torch.empty((chunk,) + tuple(src.shape[1:]), dtype=src.dtype, device=dev) for _ in range(min(n_chunks, max(1, int(depth)) + 1))]
        for b in slots:
            b.record_stream(up)
        up.wait_stream(compute)                 # the staging buffers may recycle memory the compute stream is still using
        slot_free = [None] * len(slots)         # event: the kernels that read this slot have finished
        downloaded = []                         # event per chunk: its result has reached `out` (kept only for out_frame_shape)
        for ci, i in enumerate(range(0, B, chunk)):
            s, n = ci % len(slots), min(chunk, B - i)
            host = src[i:i + n]
            if stage is not None:
                h = ci % 2
                if stage_free[h] is not None:
                    stage_free[h].synchronize()  # the upload that read this staging buffer two chunks ago has finished
                stage[h][:n].copy_(host)
                host = stage[h][:n]
            with torch.cuda.stream(up):
                if slot_free[s] is not None:
                    up.wait_event(slot_free[s])
                slots[s][:n].copy_(host, non_blocking=True)
                ev_up = torch.cuda.Event()
                ev_up.record(up)
            if stage is not None:
                stage_free[ci % 2] = ev_up
            compute.wait_event(ev_up)
            if out_frame_shape is not None and ci >= len(slots):
                downloaded[ci - len(slots)].synchronize()   # its result block is free again before fn allocates this one's
            d_out = fn(slots[s][:n], i)
            ev_done = torch.cuda.Event()
            ev_done.record(compute)
            slot_free[s] = ev_done
            down.wait_event(ev_done)
            with torch.cuda.stream(down):
                d_out.record_stream(down)
                out[i:i + n].copy_(d_out, non_blocking=True)
                if out_frame_shape is not None:
                    downloaded.append(torch.cuda.Event())
                    downloaded[-1].record(down)
            del d_out
        ev_last = torch.cuda.Event()
        ev_last.record(down)
        ev_last.synchronize()                   # the caller reads `out` on the host
        compute.wait_stream(up)
    return out


def shard_plan(n_frames, n_shards):
    """[(start, stop)] of the contiguous shards stream_frames_sharded cuts a batch into (dist.shard_range: the first shards take the
    remainder; a shard is empty when there are fewer frames than shards)."""
    return [shard_range(n_frames, k, n_shards) for k in range(n_shards)]


def stream_frames_sharded(src, make_fn, chunk, out_device, devices, out=None, out_frame_shape=None):
    """stream_frames over several CUDA devices from one process: host frames src [B,...] are cut into one contiguous shard per entry
    of `devices` (shard_plan), and each non-empty shard runs the stream_frames pipeline on its device in a host thread of its own,
    writing its slice of one shared result (pinned under stream_frames' rule).

    make_fn(device) -> fn(cuda_frames, first_frame_index) is called once per non-empty shard, in the calling thread and in shard
    order.  The index handed to fn is absolute (shard start + offset in the shard), so a fn that keys its work by the frame index
    (grain) or works per frame (everything else here) gives what one device gives.  A device may be listed more than once: its
    workers get separate upload / download streams.  Kernels go to the calling thread's current stream of each device; a pageable
    source is staged through pinned buffers of each worker's own.  An exception in a worker is raised here after every worker has
    finished, and no thread outlives the call.  One device, a CUDA source or a CUDA out_device: one stream_frames call on one
    device (CUDA batches are not sharded).  `out_frame_shape`: as stream_frames'; every worker passes it on."""
    devices = [cuda_device(d) for d in devices]
    if not devices:
        raise ValueError("vrgdg_b200: stream_frames_sharded needs at least one CUDA device")
    out_device = torch.device(out_device)
    shape_kw = {} if out_frame_shape is None else {"out_frame_shape": out_frame_shape}
    if len(devices) == 1 or src.device.type == "cuda" or out_device.type != "cpu":
        dev = src.device if src.device.type == "cuda" else devices[0]
        return stream_frames(src, make_fn(dev), chunk, out_device, dev, out=out, **shape_kw)
    src = src.contiguous()
    out_shape = _result_shape(src, out_frame_shape)
    if out is None:
        out = torch.empty(out_shape, dtype=src.dtype, pin_memory=_pin_result(src, math.prod(out_shape) * src.element_size()))
    else:
        _check_out(out, out_shape, src.dtype, out_device)
    jobs, lanes = [], {}
    for dev, (a, b) in zip(devices, shard_plan(int(src.shape[0]), len(devices))):
        if b > a:
            lane = lanes[dev] = lanes.get(dev, -1) + 1
            jobs.append((dev, lane, a, b, make_fn(dev), torch.cuda.current_stream(dev)))
    errors = [None] * len(jobs)

    def work(k, dev, lane, a, b, fn, stream):
        try:
            with torch.cuda.device(dev), torch.cuda.stream(stream):
                stream_frames(src[a:b], lambda f, i: fn(f, a + i), chunk, out_device, dev, out=out[a:b], lane=lane, **shape_kw)
        except BaseException as e:               # re-raised in the calling thread
            errors[k] = e

    threads = [threading.Thread(target=work, args=(k,) + job, name="vrgdg-shard-%d" % k) for k, job in enumerate(jobs)]
    try:
        for t in threads:
            t.start()
    finally:
        for t in threads:
            if t.ident is not None:
                t.join()
    for e in errors:
        if e is not None:
            raise e
    return out


def run_frames(images, make_fn, chunk, out_device, device, devices, out_frame_shape=None):
    """The frame loop of every node.  A host batch with a host result is sharded over `devices` (the node's devices_from_env(),
    None = not sharded) by stream_frames_sharded; anything else is the single-device stream_frames(images, make_fn(device), ...).
    make_fn(dev) -> fn(cuda_frames, absolute_first_frame) is called in the calling thread, once per non-empty shard.
    `out_frame_shape`: the shape of one result frame when fn changes it (stream_frames); None passes nothing on."""
    shape_kw = {} if out_frame_shape is None else {"out_frame_shape": out_frame_shape}
    if devices is not None and images.device.type == "cpu" and torch.device(out_device).type == "cpu":
        return stream_frames_sharded(images, make_fn, chunk, out_device, devices, **shape_kw)
    return stream_frames(images, make_fn(device), chunk, out_device, device, **shape_kw)
