"""Histogram colour match against a reference clip (frame i matched to reference frame i) without a GPU: the declaration, binding and
export of vrgdg_histmatch_apply_refs and vrgdg_histmatch_refs_scratch_bytes, the entry point's refusals, which return before any CUDA
call, and VRGDG_B200_HistogramColorMatch's refusal and per-chunk reference slicing, which come before any upload or device work."""
import ctypes
import importlib
import os
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = "vrgdg_histmatch_apply_refs"
SCRATCH = "vrgdg_histmatch_refs_scratch_bytes"


def test_entry_points_are_declared_typed_and_exported(pkg):
    nv = pkg._native
    hdr = open(os.path.join(ROOT, "include", "vrgdg_b200.h")).read()
    assert "VRGDG_API int64_t vrgdg_histmatch_refs_scratch_bytes(int B);" in hdr
    assert "VRGDG_API int vrgdg_histmatch_apply_refs(const void* in, void* out, int B, int H, int W, int dtype, const void* ref_frames,\n" \
           "                               int Hr, int Wr, float t, float one_minus_t, void* scratch, int64_t scratch_bytes, void* stream);" in hdr
    assert nv.SIGNATURES[SCRATCH] == (ctypes.c_int64, [ctypes.c_int])
    restype, argtypes = nv.SIGNATURES[ENTRY]
    assert restype is ctypes.c_int and len(argtypes) == 14
    # vrgdg_histmatch_apply's frame arguments, then the reference frames and their size, the strength, the scratch and the stream
    assert argtypes[:6] == nv.SIGNATURES["vrgdg_histmatch_apply"][1][:6]
    assert argtypes[6:] == [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p,
                            ctypes.c_int64, ctypes.c_void_p]
    nv.load_library()
    out = subprocess.run(["nm", "-D", "--defined-only", nv.LIB_PATH], capture_output=True, text=True).stdout
    for name in (ENTRY, SCRATCH):
        assert any(l.split()[-1] == name and " T " in l for l in out.splitlines()), name


def test_scratch_size_is_per_frame_and_monotone(pkg):
    lib = pkg._native.load_library()
    sizes = [int(lib.vrgdg_histmatch_refs_scratch_bytes(b)) for b in range(0, 40)]
    assert sizes[0] == 0 and all(a < b for a, b in zip(sizes, sizes[1:]))
    per_frame = sizes[1]
    assert 12 * 1024 <= per_frame <= 16 * 1024                    # counts of frame and reference plus the edge tables
    assert all(s == b * per_frame for b, s in enumerate(sizes))
    assert int(lib.vrgdg_histmatch_refs_scratch_bytes(-3)) == 0
    assert int(lib.vrgdg_histmatch_refs_scratch_bytes(1 << 20)) == (1 << 20) * per_frame    # no 32-bit overflow


def test_refusals_come_before_any_cuda_call(pkg):
    """Every case is refused with VRGDG_E_INVALID / _UNSUPPORTED / _ALIGN and a message naming the entry point; a CUDA call would
    have returned VRGDG_E_CUDA on a machine without a GPU."""
    nv = pkg._native
    lib = nv.load_library()
    src, dst, ref = ctypes.c_void_p(1 << 20), ctypes.c_void_p(2 << 20), ctypes.c_void_p(3 << 20)
    B, H, W = 3, 64, 64
    need = int(lib.vrgdg_histmatch_refs_scratch_bytes(B))
    scratch = ctypes.c_void_p(1 << 30)

    def call(B=B, H=H, W=W, dtype=nv.F32, inp=src, out=dst, frames=ref, Hr=32, Wr=48, scr=scratch, nbytes=need):
        rc = lib.vrgdg_histmatch_apply_refs(inp, out, B, H, W, dtype, frames, Hr, Wr, ctypes.c_float(1.0), ctypes.c_float(0.0), scr,
                                            ctypes.c_int64(nbytes), None)
        return rc, lib.vrgdg_last_error().decode()

    cases = [
        (dict(dtype=nv.U8BGR), nv.E_UNSUPPORTED, "uint8 frames"),
        (dict(Hr=0), nv.E_INVALID, "reference frame size 0 x 48"),
        (dict(Wr=0), nv.E_INVALID, "reference frame size 32 x 0"),
        (dict(Hr=-4, Wr=-4), nv.E_INVALID, "reference frame size"),
        (dict(Hr=1 << 16, Wr=1 << 15), nv.E_UNSUPPORTED, "exceeds 2^31"),
        (dict(dtype=7), nv.E_INVALID, "unknown dtype"),
        (dict(H=-1), nv.E_INVALID, "negative shape"),
        (dict(B=-1), nv.E_INVALID, "negative shape"),
        (dict(H=1 << 16, W=1 << 15), nv.E_UNSUPPORTED, "exceeds 2^31"),
        (dict(inp=None), nv.E_INVALID, "null frame pointer"),
        (dict(out=None), nv.E_INVALID, "null frame pointer"),
        (dict(inp=ctypes.c_void_p((1 << 20) + 2)), nv.E_ALIGN, "frame pointer not aligned"),
        (dict(frames=None), nv.E_INVALID, "null ref_frames"),
        (dict(frames=ctypes.c_void_p((3 << 20) + 2)), nv.E_ALIGN, "ref_frames not aligned"),
        (dict(scr=None), nv.E_INVALID, "null scratch"),
        (dict(scr=ctypes.c_void_p((1 << 30) + 64)), nv.E_ALIGN, "256-byte aligned"),
        (dict(nbytes=need - 1), nv.E_INVALID, "scratch too small"),
        (dict(nbytes=0), nv.E_INVALID, "scratch too small"),
    ]
    for kw, code, text in cases:
        rc, msg = call(**kw)
        assert rc == code and text in msg and ENTRY in msg, (kw, rc, msg)
    # 16-bit frames need 2-byte alignment only
    assert call(dtype=nv.F16, frames=ctypes.c_void_p((3 << 20) + 1))[0] == nv.E_ALIGN
    # an empty batch is a successful no-op before any CUDA call, whatever the pointers
    assert call(B=0, inp=None, out=None, frames=None, scr=None, nbytes=0)[0] == nv.VRGDG_OK
    assert call(H=0, frames=None, scr=None, nbytes=0)[0] == nv.VRGDG_OK
    # with valid arguments the call reaches the device query, which fails here without a GPU
    if not torch.cuda.is_available():
        assert call()[0] == nv.E_CUDA


def _fail(*a, **k):
    raise AssertionError("device work before the refusal")


def test_node_refuses_reference_batches_other_than_one_or_the_clip_before_device_work(pkg, monkeypatch):
    cn = importlib.import_module(pkg.__name__ + ".chain_nodes")
    for name in ("compute_device", "run_frames", "upload", "devices_from_env"):
        monkeypatch.setattr(cn, name, _fail)
    node = cn.VRGDG_B200_HistogramColorMatch()
    g = torch.Generator().manual_seed(3)
    x = torch.rand(3, 8, 8, 3, generator=g)
    refs = {n: torch.rand(n, 5, 7, 3, generator=g) for n in (0, 2, 4)}
    state = torch.get_rng_state()
    for n_ref, r in refs.items():
        with pytest.raises(ValueError, match=r"^reference_image batch \(%d\) must be 1 or match images batch \(3\)$" % n_ref):
            node.match_histogram(x, r, 1.0, 2)
    assert torch.equal(torch.get_rng_state(), state)             # no generator drawn from either
    # the same text as ColorMatchToReference's
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    monkeypatch.setattr(fn, "compute_device", _fail)
    with pytest.raises(ValueError) as cm_err:
        fn.ColorMatchToReference().match_color(x, refs[2], 1.0, 2)
    with pytest.raises(ValueError) as hist_err:
        node.match_histogram(x, refs[2], 1.0, 2)
    assert str(hist_err.value) == str(cm_err.value)


class _FakeOps:
    """stands in for ops: records the calls the node makes"""

    def __init__(self):
        self.calls = []
        fake = self

        class Counts:
            def to(self, card):
                fake.calls.append(("counts_to", card))
                return self
        self.Counts = Counts

    def hist_counts(self, t):
        self.calls.append(("hist_counts", t.clone()))
        return self.Counts()

    def histmatch_tables(self, fc, rc):
        self.calls.append(("histmatch_tables",))
        return "tables"

    def histmatch_apply(self, frames, tables, t, omt):
        self.calls.append(("histmatch_apply",))
        return frames.clone()

    def histmatch_apply_refs(self, frames, refs, t, omt, scratch=None):
        self.calls.append(("histmatch_apply_refs", refs.clone(), frames.dtype, t, omt, scratch))
        return frames.clone(), "scratch"


class _NoDevice:
    def __init__(self, dev):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _node_on_fakes(pkg, monkeypatch):
    cn = importlib.import_module(pkg.__name__ + ".chain_nodes")
    ops_mod = importlib.import_module(pkg.__name__ + ".ops")
    fake = _FakeOps()
    for name in ("hist_counts", "histmatch_tables", "histmatch_apply", "histmatch_apply_refs"):
        monkeypatch.setattr(ops_mod, name, getattr(fake, name))
    seen = {}

    def run_frames(images, make_fn, chunk, out_device, device, devices):
        run = make_fn(device)
        seen["chunks"] = [(i, min(i + chunk, images.shape[0])) for i in range(0, images.shape[0], chunk)]
        return torch.cat([run(images[a:b], a) for a, b in seen["chunks"]])

    monkeypatch.setattr(cn, "run_frames", run_frames)
    monkeypatch.setattr(cn, "compute_device", lambda images=None: torch.device("cpu"))
    monkeypatch.setattr(cn, "devices_from_env", lambda: None)
    monkeypatch.setattr(cn, "upload", lambda t, dev: t.clone())
    monkeypatch.setattr(torch.cuda, "device", _NoDevice)
    return cn.VRGDG_B200_HistogramColorMatch(), fake, seen


def test_node_uploads_only_each_chunks_reference_frames(pkg, monkeypatch):
    """n_ref == B: no whole-clip counts; chunk [first, first + n) gets reference_image[first:first + n] in the frames' dtype through
    one histmatch_apply_refs call, and the worker's scratch is handed from call to call"""
    node, fake, seen = _node_on_fakes(pkg, monkeypatch)
    x = torch.rand(7, 4, 4, 3, dtype=torch.bfloat16)
    refs = torch.rand(7, 3, 5, 3)
    node.match_histogram(x, refs, 0.35, 3)
    assert seen["chunks"] == [(0, 3), (3, 6), (6, 7)]
    assert [c[0] for c in fake.calls] == ["histmatch_apply_refs"] * 3
    for (name, got, dtype, t, omt, scratch), (a, b), prev in zip(fake.calls, seen["chunks"], (None, "scratch", "scratch")):
        assert dtype == torch.bfloat16 and torch.equal(got, refs[a:b].to(torch.bfloat16)) and scratch == prev
        assert t == 0.35 and omt == 1.0 - 0.35


def test_node_keeps_the_single_reference_path(pkg, monkeypatch):
    """n_ref == 1 (also when B == 1): the reference is counted once, in the frames' dtype, and its counts are copied to the card;
    each chunk then makes its tables and the apply pass"""
    node, fake, seen = _node_on_fakes(pkg, monkeypatch)
    x = torch.rand(5, 4, 4, 3, dtype=torch.float16)
    one = torch.rand(1, 3, 5, 3)
    node.match_histogram(x, one, 0.5, 2)
    names = [c[0] for c in fake.calls]
    assert names[:2] == ["hist_counts", "counts_to"] and torch.equal(fake.calls[0][1], one.half())
    assert names[2:] == ["hist_counts", "histmatch_tables", "histmatch_apply"] * 3
    fake.calls.clear()
    node.match_histogram(x[:1], one, 0.5, 2)
    assert "histmatch_apply_refs" not in [c[0] for c in fake.calls]
