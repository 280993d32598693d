"""Device policy and host<->device frame streaming shared by the node classes."""
import torch


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


def _side_streams(dev):
    """(upload, download) streams of a device, created once (stream creation is not free and ComfyUI calls nodes repeatedly)."""
    key = (dev.type, dev.index)
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


def stream_frames(src, fn, chunk, out_device, device=None, out=None, depth=2):
    """Apply fn(cuda_frames, first_frame_index) -> cuda_frames over src [B,...] in chunks of `chunk` frames (0 / None = all).

    CUDA input: chunked as well (the reference bounds device memory with its batch_size widget the same way, nodes.py:49-62);
    one call when the chunk covers the batch.  CPU input: a three-stream pipeline - chunk k+1.. are uploaded into `depth`+1
    reusable staging buffers while chunk k computes and earlier results download; only the last download is waited for.
    Pinned source / result tensors make the copies truly asynchronous (the result is pinned when the source is).  `out`:
    optional preallocated result on out_device (reused across calls so that pinning cost is paid once)."""
    B = int(src.shape[0])
    out_device = torch.device(out_device)
    chunk = B if chunk is None or int(chunk) <= 0 else min(int(chunk), max(B, 1))
    if src.device.type == "cuda":
        if chunk >= B:
            res = fn(src, 0)
            return res if res.device == out_device else res.to(out_device)
        to_host = out_device.type == "cpu"
        res = torch.empty(src.shape, dtype=src.dtype, device=out_device, pin_memory=to_host and _pin_result(src, src.numel() * src.element_size()))
        for i in range(0, B, chunk):
            res[i:i + chunk].copy_(fn(src[i:i + chunk], i), non_blocking=to_host)
        if to_host:
            torch.cuda.current_stream(src.device).synchronize()
        return res
    dev = device if device is not None else compute_device()
    if B == 0:
        return torch.empty_like(src, device=out_device)
    src = src.contiguous()
    to_cpu = out_device.type == "cpu"
    # Host frames move in pipeline chunks of at most VRGDG_STREAM_CHUNK_BYTES (default 256 MiB, at least one frame): a chunk as large
    # as the batch would serialise upload, kernels and download.  Every caller's fn is independent of how the batch is cut (noise is
    # keyed by the absolute frame index, statistics are per frame, temporal neighbours are fetched by index).
    chunk = pipeline_chunk(chunk, src[0].numel() * src.element_size())
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
        up, down = _side_streams(dev)
        if out is None:
            out = torch.empty(src.shape, dtype=src.dtype, pin_memory=_pin_result(src, src.numel() * src.element_size())) if to_cpu \
                else torch.empty(src.shape, dtype=src.dtype, device=out_device)
        elif out.shape != src.shape or out.dtype != src.dtype or out.device != out_device:
            raise ValueError("vrgdg_b200: `out` must match the source frames in shape and dtype and live on %s" % out_device)
        n_chunks = (B + chunk - 1) // chunk
        slots = [torch.empty((chunk,) + tuple(src.shape[1:]), dtype=src.dtype, device=dev) for _ in range(min(n_chunks, max(1, int(depth)) + 1))]
        for b in slots:
            b.record_stream(up)
        up.wait_stream(compute)                 # the staging buffers may recycle memory the compute stream is still using
        slot_free = [None] * len(slots)         # event: the kernels that read this slot have finished
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
            d_out = fn(slots[s][:n], i)
            ev_done = torch.cuda.Event()
            ev_done.record(compute)
            slot_free[s] = ev_done
            down.wait_event(ev_done)
            with torch.cuda.stream(down):
                d_out.record_stream(down)
                out[i:i + n].copy_(d_out, non_blocking=True)
            del d_out
        ev_last = torch.cuda.Event()
        ev_last.record(down)
        ev_last.synchronize()                   # the caller reads `out` on the host
        compute.wait_stream(up)
    return out
