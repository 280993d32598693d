"""Fused post-processing chain: grain -> colour match -> 3D LUT -> 3x3 stencil -> post grain in ONE pass over HBM.

Semantics = the reference nodes applied one after another (FastFilmGrain nodes.py:41-66 ->
ColorMatchToReference :91-124 -> VRGDG_LUTS VRGDG_IV_Adjustments.py:345-361 -> FastUnsharpSharpen nodes.py:156-209),
or the standalone enhancer's unsharp -> seeded grain (_apply_effects_batch,
VRGDG_StandaloneVideoEnhancerNodes.py:278-294) via `post_grain`.  Any subset of stages may be enabled.
RGBA frames take the subset the reference defines on 4 channels: LUT -> NumPy-path stencil (PostChain.check_frames).
"""
import ctypes

import torch

from . import _native as nv
from . import ops
from ._runtime import compute_device, cuda_device, pipeline_chunk, stream_frames, stream_frames_sharded, upload


class PostChain:
    def __init__(self, grain=None, colormatch=None, lut=None, stencil=None, post_grain=None, device=None, devices=None):
        """
        grain / post_grain: dict(intensity, saturation_mix, seed, seed_mode=SEED_PER_CLIP); post_grain also takes
                            seed_mode=SEED_TORCH_PER_FRAME (torch's CUDA randn stream of the enhancer's per-frame seeded generators)
        grain may instead carry torch_global=dict(seed, philox_offset, clip_frames, draw_frames): a snapshot of a global CUDA
                            generator (filter_nodes.GlobalStreamDraws), so that the grain is FastFilmGrain's under
                            VRGDG_GRAIN_NOISE=torch_cuda: one randn_like per draw_frames frames of a clip of clip_frames frames.
                            The chain neither reads nor advances a generator; the frames' first_frame keys the draws.
        colormatch:         dict(reference_image=[1,H,W,3] tensor  |  reference_frames=[N,Hr,Wr,3] tensor  |  ref_sums=[1|N,7] float64,
                            strength).  reference_frames / ref_sums with N > 1 are a reference CLIP: frame f of the clip (absolute
                            index, first_frame + i) is matched to reference frame f, at every chunk size (ColorMatchToReference's
                            pairing); a call whose frames reach past frame N - 1 raises ValueError before any device work.  Each
                            call uploads only the reference frames of its own indices (host or CUDA, any size and float dtype; they
                            are converted to the frames' dtype on the frames' card).  One reference frame is broadcast.
        lut:                dict(lut_data={"lut","domain_min","domain_max"}, strength 0..10)
        stencil:            dict(op=STENCIL_*, strength, border=BORDER_REPLICATE)
        devices:            CUDA devices run_host shards host batches over (default None: `device` alone).  The first one is `device`;
                            a device may be listed twice (two workers on one card).
        """
        if devices is None:
            self.device = torch.device(device) if device is not None else compute_device()
            self.devices = [self.device]
        else:
            self.devices = [cuda_device(d) for d in devices]
            if not self.devices:
                raise ValueError("vrgdg_b200: PostChain(devices=...) needs at least one CUDA device")
            if device is not None and cuda_device(device) != self.devices[0]:
                raise ValueError("vrgdg_b200: PostChain(device=%s) is not the first of devices=%s" % (device, self.devices))
            self.device = self.devices[0]
        self.grain, self.colormatch, self.lut, self.stencil, self.post_grain = grain, colormatch, lut, stencil, post_grain
        # per device: the packed LUT and the reference statistics (made on `device`, copied to the others); per (device, worker on
        # that device): the colour-match scratch
        self._luts, self._refs, self._scratch = {}, {}, {}
        self._ref_frames = None     # the reference clip (reference_frames with more than one frame), where the caller keeps it
        self.timing = None          # set to a list to collect (moments_start, moments_end, apply_start, apply_end) CUDA events per call
        # colour-match schedule (vrgdg_chain_cm_apply): one library call; `split` = the three-call path (statistics, parameters,
        # apply as separate entry points; what `timing` needs), `recompute` / `group_frames`: see include/vrgdg_b200.h
        self.split, self.recompute, self.group_frames, self.serial = False, False, 0, False
        if lut is not None:
            packed = ops.pack_lut(lut["lut_data"]["lut"], self.device)
            self._luts = {dev: packed if dev == self.device else ops.PackedLut(packed.data.to(dev), packed.size)
                          for dev in dict.fromkeys(self.devices)}
        if colormatch is not None:
            frames = colormatch.get("reference_frames")
            if frames is not None:
                if not isinstance(frames, torch.Tensor) or frames.ndim != 4 or frames.shape[-1] != 3 or frames.shape[0] < 1:
                    raise ValueError("vrgdg_b200: PostChain colormatch reference_frames must be a tensor [N,H,W,3] with N >= 1")
                if colormatch.get("reference_image") is not None or colormatch.get("ref_sums") is not None:
                    raise ValueError("vrgdg_b200: PostChain colormatch takes one of reference_image, reference_frames, ref_sums")
            if frames is not None and frames.shape[0] > 1:
                self._ref_frames = frames
            else:
                self.set_reference(colormatch.get("reference_image") if frames is None else frames, colormatch.get("ref_sums"))

    # -- colour-match reference statistics (the only cross-rank quantity, see dist.py) --
    def set_reference(self, reference_image=None, ref_sums=None):
        """The statistics are made once, on `device`, and copied to the other devices: a copy is bit-identical to a recomputation and
        does not read the reference image once per GPU."""
        if ref_sums is not None:
            sums = ref_sums.to(self.device, torch.float64).reshape(-1, 7).contiguous()
        elif reference_image is not None:
            sums = ops.lab_moments(upload(reference_image, self.device))
        else:
            raise ValueError("colour match needs reference_image or ref_sums")
        self._refs = {dev: sums if dev == self.device else sums.to(dev) for dev in dict.fromkeys(self.devices)}
        self._ref_frames = None

    def _n_ref(self):
        """frames in the reference: 1 (broadcast) or the length of a reference clip; None without colour match"""
        if self.colormatch is None:
            return None
        return int(self._ref_frames.shape[0]) if self._ref_frames is not None else int(self._ref_sums.shape[0])

    def check_reference(self, n_frames, first_frame):
        """A reference clip pairs by absolute frame index: frames [first_frame, first_frame + n_frames) need as many reference frames.
        ValueError otherwise, before any device work."""
        n_ref = self._n_ref()
        if n_ref is not None and n_ref != 1 and int(first_frame) + int(n_frames) > n_ref:
            raise ValueError("vrgdg_b200: PostChain colour match has a reference clip of %d frames, but the frames are [%d, %d) of the clip"
                             % (n_ref, int(first_frame), int(first_frame) + int(n_frames)))

    def _reference_for(self, frames, first_frame):
        """(reference frames, None) or (None, reference sums) for frames [first_frame, first_frame + B) on frames.device: the
        reference clip's frames of those indices, uploaded and converted to the frames' dtype there, or the sums' rows"""
        B = int(frames.shape[0])
        if self._ref_frames is not None:
            return upload(self._ref_frames[first_frame:first_frame + B], frames.device).to(frames.dtype), None
        sums = self._on(self._refs, frames.device)
        return None, (sums if sums.shape[0] == 1 else sums[first_frame:first_frame + B])

    @property
    def _ref_sums(self):
        """the reference statistics on `device`"""
        return self._refs.get(self.device)

    @staticmethod
    def _on(table, dev):
        """The copy in `table` for frames on `dev`.  A single-device chain has one copy, used whatever the frames' device."""
        if len(table) == 1:
            return next(iter(table.values()))
        if dev not in table:
            raise ValueError("vrgdg_b200: frames on %s, but this PostChain runs on %s" % (dev, list(table)))
        return table[dev]

    def _desc(self, frames, first_frame, keep, ext_noise=None, fused_cm=False):
        d = nv.ChainDesc()
        if self.grain is not None:
            s = float(self.grain["saturation_mix"])
            d.grain_enabled = 1
            d.grain_intensity, d.grain_sat, d.grain_one_minus_sat = float(self.grain["intensity"]), s, 1.0 - s
            d.grain_seed = int(self.grain.get("seed", 0)) & 0xFFFFFFFFFFFFFFFF
            d.grain_frame0 = int(first_frame)
            d.grain_seed_mode = int(self.grain.get("seed_mode", nv.SEED_PER_CLIP))
        if self.lut is not None:
            data = self.lut["lut_data"]
            blend = max(0.0, min(10.0, float(self.lut.get("strength", 10.0)))) / 10.0
            if blend > 0.0:
                fdt = torch.float32 if frames.dtype == torch.uint8 else frames.dtype     # uint8 frames become float32 tensors in the reference
                dmin = data["domain_min"].to(dtype=fdt)
                span = torch.clamp(data["domain_max"].to(dtype=fdt) - dmin, min=1e-6)
                d.lut_enabled = 1
                packed = self._on(self._luts, frames.device)
                d.lut = packed.data.data_ptr()
                d.lut_size = packed.size
                d.lut_dmin = (ctypes.c_float * 3)(*dmin.float().tolist())
                d.lut_dspan = (ctypes.c_float * 3)(*span.float().tolist())
                d.lut_blend, d.lut_one_minus_blend = blend, 1.0 - blend
        if self.stencil is not None and not (self.stencil["op"] == nv.STENCIL_NONE):
            d.stencil_op = int(self.stencil["op"])
            d.stencil_strength = float(self.stencil["strength"])
            d.stencil_border = int(self.stencil.get("border", nv.BORDER_REPLICATE))
        if self.post_grain is not None:
            s = float(self.post_grain["saturation_mix"])
            d.post_grain_enabled = 1
            d.post_intensity, d.post_sat, d.post_one_minus_sat = float(self.post_grain["intensity"]), s, 1.0 - s
            d.post_seed = int(self.post_grain.get("seed", 0)) & 0xFFFFFFFFFFFFFFFF
            d.post_frame0 = int(first_frame)
            d.post_seed_mode = int(self.post_grain.get("seed_mode", nv.SEED_PER_FRAME))
        if self.colormatch is not None and fused_cm:
            t = float(self.colormatch.get("strength", 1.0))
            d.colormatch_enabled = 1
            d.cm_t, d.cm_one_minus_t = t, 1.0 - t
        elif self.colormatch is not None:
            # per-frame LAB moments of the colour-match INPUT (= grain output when grain is enabled): a first pass
            # that recomputes the counter-based grain instead of materialising it
            ref, ref_sums = self._reference_for(frames, first_frame)
            if ref is not None:
                ref_sums = ops.lab_moments(ref)
                del ref
            if self.timing is not None:
                self._ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                self._ev[0].record()
            sums = ops.chain_lab_moments(frames, d, ext_noise=ext_noise)
            params = ops.colormatch_params(sums, ref_sums)
            if self.timing is not None:
                self._ev[1].record()
            keep.append(params)
            t = float(self.colormatch.get("strength", 1.0))
            d.colormatch_enabled = 1
            d.cm_params = params.data_ptr()
            d.cm_t, d.cm_one_minus_t = t, 1.0 - t
        return d

    def check_frames(self, frames):
        """RGBA frames [B,H,W,4] take the stages the reference defines on 4 channels: `lut` (RGB graded, alpha carried) and the
        NumPy-path `stencil` ops (every channel filtered).  Anything else on RGBA raises ValueError here, before any device work."""
        if not (isinstance(frames, torch.Tensor) and frames.ndim == 4 and frames.shape[-1] == 4):
            return
        for name in ("grain", "colormatch", "post_grain"):
            if getattr(self, name) is not None:
                raise ValueError("vrgdg_b200: PostChain stage `%s` takes 3-channel frames, got 4 channels (RGBA frames take `lut` and "
                                 "`stencil` only)" % name)
        if self.stencil is not None and self.stencil["op"] in (nv.STENCIL_LAPLACIAN_GPU, nv.STENCIL_SOBEL_GPU):
            raise ValueError("vrgdg_b200: PostChain stencil op %d (a torch conv2d path) takes 3-channel frames, got 4 channels"
                             % self.stencil["op"])

    def _torch_global(self, frames, ext_noise):
        """the grain's global-stream snapshot, or None; ValueError for what that stream cannot grain (uint8 frames, whose draws the
        reference makes from fp32 tensors, and a caller's ext_noise, which would replace the stream)"""
        tg = self.grain.get("torch_global") if self.grain is not None else None
        if tg is None:
            return None
        if ext_noise is not None:
            raise ValueError("vrgdg_b200: PostChain grain with torch_global draws its own noise; ext_noise cannot replace it")
        if isinstance(frames, torch.Tensor) and frames.dtype == torch.uint8:
            raise ValueError("vrgdg_b200: PostChain grain with torch_global takes float frames (IMAGE tensors), got uint8")
        return tg

    def __call__(self, frames, first_frame=0, ext_noise=None, out=None, fast_math=False):
        """frames: CUDA [B,H,W,3], or [B,H,W,4] with only `lut` / `stencil` set (check_frames); first_frame: absolute index of
        frames[0] in the clip (keys the grain).  ext_noise (tests): N(0,1) tensor replacing the generator; fast_math then selects the
        production arithmetic."""
        return self._run(frames, first_frame, 0, ext_noise, out, fast_math)

    def _run(self, frames, first_frame, worker, ext_noise=None, out=None, fast_math=False):
        """__call__ with the colour-match scratch of `worker` (the index of a stream_frames_sharded worker on the frames' device)."""
        self.check_frames(frames)
        self.check_reference(frames.shape[0], first_frame)
        tg = self._torch_global(frames, ext_noise)
        if tg is None:
            return self._apply(frames, first_frame, worker, ext_noise, out, fast_math)
        # the global stream's noise, materialised for at most one pipeline chunk of frames at a time (results are per frame), then the
        # external-noise chain with the reference's op order
        B = int(frames.shape[0])
        sub = B if B == 0 else pipeline_chunk(B, frames[0].numel() * frames.element_size())
        if sub >= B:
            noise = ops.grain_noise_torch_global(frames, tg["seed"], tg["philox_offset"], first_frame, tg["clip_frames"], tg["draw_frames"])
            return self._apply(frames, first_frame, worker, noise, out, False)
        out = torch.empty_like(frames) if out is None else out
        for i in range(0, B, sub):
            f = frames[i:i + sub]
            noise = ops.grain_noise_torch_global(f, tg["seed"], tg["philox_offset"], first_frame + i, tg["clip_frames"], tg["draw_frames"])
            self._apply(f, first_frame + i, worker, noise, out[i:i + sub], False)
            del noise
        return out

    def _apply(self, frames, first_frame, worker, ext_noise, out, fast_math):
        """_run on the chain's own noise source or on ext_noise"""
        keep = []
        if self.colormatch is not None and not self.split and self.timing is None:
            d = self._desc(frames, first_frame, keep, ext_noise, fused_cm=True)
            key = (frames.device, worker)
            ref, ref_sums = self._reference_for(frames, first_frame)
            if ref is not None:
                res, self._scratch[key] = ops.chain_cm_apply_refs(frames, d, ref, ext_noise=ext_noise, out=out, fast_math=fast_math,
                                                                  recompute=self.recompute, group_frames=self.group_frames,
                                                                  scratch=self._scratch.get(key), serial=self.serial)
                return res
            res, self._scratch[key] = ops.chain_cm_apply(frames, d, ref_sums, ext_noise=ext_noise, out=out,
                                                         fast_math=fast_math, recompute=self.recompute, group_frames=self.group_frames,
                                                         scratch=self._scratch.get(key), serial=self.serial)
            return res
        d = self._desc(frames, first_frame, keep, ext_noise)
        if self.timing is None:
            return ops.chain_apply(frames, d, ext_noise=ext_noise, keepalive=keep, out=out, fast_math=fast_math)
        ev = getattr(self, "_ev", None) if self.colormatch is not None else None
        if ev is None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            ev[1].record()
        ev[2].record()
        res = ops.chain_apply(frames, d, ext_noise=ext_noise, keepalive=keep, out=out, fast_math=fast_math)
        ev[3].record()
        self.timing.append(tuple(ev))
        self._ev = None
        return res

    def make_fn(self, first_frame=0):
        """make_fn of _runtime.stream_frames_sharded for this chain: every worker gets fn(frames, i) = self(frames, first_frame + i)
        with a colour-match scratch of its own, so that two workers on one card never share one.  `first_frame`: absolute index of
        the batch's first frame in the clip."""
        if self.timing is not None:
            raise ValueError("vrgdg_b200: PostChain.timing is collected by single-device calls only")
        workers = {}

        def make(dev):
            k = workers[dev] = workers.get(dev, -1) + 1
            return lambda f, i: self._run(f, first_frame + i, k)
        return make

    def run_host(self, frames_cpu, chunk_frames=8, first_frame=0, out=None):
        """Host frames in, host frames out: chunked upload / compute / download on three streams.  Pass pinned tensors
        (and a reusable pinned `out`) for asynchronous copies.  With several `devices` the batch is cut into one contiguous shard per
        device, each streamed by its own host thread into its slice of one result (stream_frames_sharded); the result is
        bit-identical to one device's."""
        self.check_frames(frames_cpu)
        self.check_reference(frames_cpu.shape[0], first_frame)
        self._torch_global(frames_cpu, None)
        if len(self.devices) == 1:
            return stream_frames(frames_cpu, lambda f, i: self(f, first_frame + i), chunk_frames, torch.device("cpu"), self.device, out=out)
        return stream_frames_sharded(frames_cpu, self.make_fn(first_frame), chunk_frames, torch.device("cpu"), self.devices, out=out)
