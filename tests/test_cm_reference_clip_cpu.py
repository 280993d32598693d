"""Colour match against a reference clip (frame i matched to reference frame i) without a GPU: the declaration, binding and export of
vrgdg_chain_cm_apply_refs, its refusals, which return before any CUDA call, and the refusals and per-chunk reference slicing of
ColorMatchToReference, PostChain and VRGDG_B200_PostChain, which come before any upload or device work."""
import ctypes
import importlib
import os
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = "vrgdg_chain_cm_apply_refs"


def test_entry_point_is_declared_typed_and_exported(pkg):
    nv = pkg._native
    hdr = open(os.path.join(ROOT, "include", "vrgdg_b200.h")).read()
    assert "VRGDG_API int vrgdg_chain_cm_apply_refs(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc,\n" \
           "                              const void* ref_frames, int Hr, int Wr, double* ref_sums, const void* ext_noise, int flags," in hdr
    restype, argtypes = nv.SIGNATURES[ENTRY]
    assert restype is ctypes.c_int and len(argtypes) == 17
    # everything vrgdg_chain_cm_apply takes, ref_sums / n_ref replaced by ref_frames, Hr, Wr, ref_sums
    base = nv.SIGNATURES["vrgdg_chain_cm_apply"][1]
    assert argtypes[:7] == base[:7] and argtypes[11:] == base[9:]
    assert argtypes[7:11] == [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    nv.load_library()
    out = subprocess.run(["nm", "-D", "--defined-only", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert any(l.split()[-1] == ENTRY and " T " in l for l in out.splitlines())


def _cm_desc(nv, **kw):
    d = nv.ChainDesc()
    d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, 1.0, 0.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_refusals_come_before_any_cuda_call(pkg):
    """Every case is refused with VRGDG_E_INVALID / _UNSUPPORTED / _ALIGN and a message naming the entry point; a CUDA call would
    have returned VRGDG_E_CUDA on a machine without a GPU.  The cases vrgdg_chain_cm_apply also refuses give its message."""
    nv = pkg._native
    lib = nv.load_library()
    src, dst, ref, sums = ctypes.c_void_p(1 << 20), ctypes.c_void_p(2 << 20), ctypes.c_void_p(3 << 20), ctypes.c_void_p(4 << 20)
    B, H, W = 3, 64, 64
    need = int(lib.vrgdg_chain_cm_scratch_bytes(B, H, W, nv.F32, 0, 0))
    scratch = ctypes.c_void_p(1 << 30)
    cm = _cm_desc(nv)

    def refs(desc=cm, B=B, H=H, W=W, dtype=nv.F32, inp=src, out=dst, frames=ref, Hr=32, Wr=48, ref_sums=sums, scr=scratch, nbytes=need):
        rc = lib.vrgdg_chain_cm_apply_refs(inp, out, B, H, W, dtype, ctypes.byref(desc) if desc is not None else None, frames, Hr, Wr,
                                           ref_sums, None, 0, scr, ctypes.c_int64(nbytes), 0, None)
        return rc, lib.vrgdg_last_error().decode()

    def one_call(desc=cm, B=B, H=H, W=W, dtype=nv.F32, inp=src, out=dst, ref_sums=sums, scr=scratch, nbytes=need, **_):
        rc = lib.vrgdg_chain_cm_apply(inp, out, B, H, W, dtype, ctypes.byref(desc) if desc is not None else None, ref_sums, B, None, 0,
                                      scr, ctypes.c_int64(nbytes), 0, None)
        return rc, lib.vrgdg_last_error().decode()

    own = [
        (dict(dtype=nv.U8BGR), nv.E_UNSUPPORTED, "uint8 frames"),
        (dict(Hr=0), nv.E_INVALID, "reference frame size 0 x 48"),
        (dict(Wr=0), nv.E_INVALID, "reference frame size 32 x 0"),
        (dict(Hr=-4, Wr=-4), nv.E_INVALID, "reference frame size"),
        (dict(Hr=1 << 16, Wr=1 << 15), nv.E_UNSUPPORTED, "exceeds 2^31"),
        (dict(frames=None), nv.E_INVALID, "null ref_frames"),
        (dict(frames=ctypes.c_void_p((3 << 20) + 2)), nv.E_ALIGN, "ref_frames not aligned"),
        (dict(ref_sums=ctypes.c_void_p((4 << 20) + 4)), nv.E_ALIGN, "ref_sums must be 8-byte aligned"),
    ]
    shared = [
        (dict(desc=None), nv.E_INVALID, "null descriptor"),
        (dict(desc=nv.ChainDesc()), nv.E_INVALID, "no colour-match stage"),
        (dict(dtype=7), nv.E_INVALID, "unknown dtype"),
        (dict(H=-1), nv.E_INVALID, "negative shape"),
        (dict(inp=None), nv.E_INVALID, "null frame pointer"),
        (dict(ref_sums=None), nv.E_INVALID, "null pointer"),
        (dict(scr=None), nv.E_INVALID, "null pointer"),
        (dict(out=src), nv.E_INVALID, "cannot run in place"),
        (dict(scr=ctypes.c_void_p((1 << 30) + 64)), nv.E_ALIGN, "256-byte aligned"),
        (dict(nbytes=need - 1), nv.E_INVALID, "scratch too small"),
        (dict(desc=_cm_desc(nv, grain_enabled=1, grain_seed_mode=nv.SEED_TORCH_PER_FRAME)), nv.E_UNSUPPORTED, "torch-stream modes"),
        (dict(desc=_cm_desc(nv, grain_enabled=1, grain_seed_mode=9)), nv.E_INVALID, "bad grain seed_mode 9"),
    ]
    for kw, code, text in own + shared:
        rc, msg = refs(**kw)
        assert rc == code and text in msg and ENTRY in msg, (kw, rc, msg)
    for kw, code, text in shared:
        rc, msg = one_call(**kw)
        assert (rc, msg.replace("vrgdg_chain_cm_apply", ENTRY)) == refs(**kw), kw
    # an empty batch is a successful no-op before any CUDA call, whatever the pointers
    assert refs(B=0, inp=None, out=None, frames=None, ref_sums=None, scr=None, nbytes=0)[0] == nv.VRGDG_OK
    assert refs(H=0, frames=None)[0] == nv.VRGDG_OK


def _fail(*a, **k):
    raise AssertionError("device work before the refusal")


def test_postchain_refuses_a_reference_clip_that_does_not_cover_the_frames_before_any_upload(pkg, monkeypatch):
    chain_mod = importlib.import_module(pkg.__name__ + ".chain")
    monkeypatch.setattr(chain_mod, "upload", _fail)
    monkeypatch.setattr(chain_mod, "stream_frames", _fail)
    monkeypatch.setattr(chain_mod, "stream_frames_sharded", _fail)
    refs = torch.rand(5, 4, 6, 3)
    chain = pkg.chain.PostChain(colormatch=dict(reference_frames=refs, strength=1.0), device="cuda:0")
    for frames, first in ((torch.rand(6, 8, 8, 3), 0), (torch.rand(2, 8, 8, 3), 4), (torch.rand(1, 8, 8, 3), 5)):
        with pytest.raises(ValueError, match=r"reference clip of 5 frames, but the frames are \[%d, %d\)" % (first, first + len(frames))):
            chain(frames, first_frame=first)
        with pytest.raises(ValueError, match="reference clip of 5 frames"):
            chain.run_host(frames, first_frame=first)
    with pytest.raises(ValueError, match="reference clip of 5 frames"):
        chain.make_fn(4)(torch.device("cuda:0"))(torch.rand(3, 8, 8, 3), 0)
    # a reference clip on an RGBA batch: the colour-match stage takes 3 channels
    with pytest.raises(ValueError, match="stage `colormatch` takes 3-channel frames"):
        chain(torch.rand(5, 8, 8, 4))
    with pytest.raises(ValueError, match="stage `colormatch` takes 3-channel frames"):
        chain.run_host(torch.rand(5, 8, 8, 4))
    # malformed specs
    for bad in (torch.rand(5, 4, 6, 4), torch.rand(4, 6, 3), torch.rand(0, 4, 6, 3)):
        with pytest.raises(ValueError, match="reference_frames must be a tensor"):
            pkg.chain.PostChain(colormatch=dict(reference_frames=bad), device="cuda:0")
    with pytest.raises(ValueError, match="one of reference_image, reference_frames, ref_sums"):
        pkg.chain.PostChain(colormatch=dict(reference_frames=refs, reference_image=refs[:1]), device="cuda:0")


class _Recorder:
    """stands in for PostChain: records the colour-match spec the node hands over"""

    def __init__(self):
        self.specs = []

    def chain(self, colormatch=None, **kw):
        self.specs.append(colormatch)

        class C:
            device = torch.device("cpu")

            def make_fn(self):
                return None
        return C()


def test_node_refuses_reference_batches_other_than_one_or_the_clip_before_device_work(pkg, monkeypatch):
    cn = importlib.import_module(pkg.__name__ + ".chain_nodes")
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    for mod in (cn, fn):
        monkeypatch.setattr(mod, "compute_device", _fail)
        monkeypatch.setattr(mod, "run_frames", _fail)
    monkeypatch.setattr(cn, "PostChain", _fail)
    node, cm_node = cn.VRGDG_B200_PostChain(), fn.ColorMatchToReference()
    x = torch.rand(3, 8, 8, 3)
    for n_ref in (2, 4):
        refs = torch.rand(n_ref, 5, 7, 3)
        want = r"reference_image batch \(%d\) must be 1 or match images batch \(3\)" % n_ref
        with pytest.raises(ValueError, match=want):
            node.apply_chain(x, 0.04, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 2, reference_image=refs)
        with pytest.raises(ValueError, match=want):
            cm_node.match_color(x, refs, 1.0, 2)
    # RGBA batches keep their refusal of any reference
    with pytest.raises(ValueError, match="reference_image \\(colour match\\) takes 3-channel images"):
        node.apply_chain(torch.rand(3, 8, 8, 4), 0.0, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 2, reference_image=torch.rand(3, 8, 8, 3))


def test_node_hands_one_reference_as_today_and_a_clip_as_reference_frames(pkg, monkeypatch):
    cn = importlib.import_module(pkg.__name__ + ".chain_nodes")
    rec = _Recorder()
    monkeypatch.setattr(cn, "PostChain", rec.chain)
    monkeypatch.setattr(cn, "compute_device", lambda images=None: torch.device("cpu"))
    monkeypatch.setattr(cn, "run_frames", lambda images, *a: images.clone())
    node = cn.VRGDG_B200_PostChain()
    x = torch.rand(3, 8, 8, 3, dtype=torch.float16)
    one, clip = torch.rand(1, 5, 7, 3), torch.rand(3, 5, 7, 3)
    node.apply_chain(x, 0.0, 0.5, 0.7, "none", 10.0, "none", 0.5, False, 2, reference_image=one)
    assert set(rec.specs[-1]) == {"reference_image", "strength"} and rec.specs[-1]["strength"] == 0.7
    assert torch.equal(rec.specs[-1]["reference_image"], one.half())
    node.apply_chain(x, 0.0, 0.5, 0.7, "none", 10.0, "none", 0.5, False, 2, reference_image=clip)
    assert set(rec.specs[-1]) == {"reference_frames", "strength"}
    assert rec.specs[-1]["reference_frames"] is clip            # not converted or copied: each chunk uploads its own frames


def test_colormatch_node_uploads_only_each_chunks_reference_frames(pkg, monkeypatch):
    """n_ref == B: no whole-clip statistics; chunk [first, first + n) gets reference_image[first:first + n] in the frames' dtype,
    through one chain_cm_apply_refs call, and the worker's scratch is handed from call to call"""
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    calls = []

    class FakeOps:
        @staticmethod
        def lab_moments(t):
            calls.append(("lab_moments",))

        @staticmethod
        def chain_cm_apply(frames, d, rs, scratch=None):
            calls.append(("chain_cm_apply",))

        @staticmethod
        def chain_cm_apply_refs(frames, d, refs, scratch=None):
            calls.append(("chain_cm_apply_refs", refs.clone(), frames.dtype, scratch))
            return frames.clone(), "scratch"

    def run_frames(images, make_fn, chunk, out_device, device, devices):
        run = make_fn(device)
        return torch.cat([run(images[i:i + chunk], i) for i in range(0, images.shape[0], chunk)])

    monkeypatch.setattr(fn, "ops", FakeOps)
    monkeypatch.setattr(fn, "run_frames", run_frames)
    monkeypatch.setattr(fn, "compute_device", lambda images=None: torch.device("cpu"))
    monkeypatch.setattr(fn, "upload", lambda t, dev: t.clone())
    x = torch.rand(7, 4, 4, 3, dtype=torch.bfloat16)
    refs = torch.rand(7, 3, 5, 3)
    fn.ColorMatchToReference().match_color(x, refs, 1.0, 3)
    assert [c[0] for c in calls] == ["chain_cm_apply_refs"] * 3
    for (name, got, dtype, scratch), (a, b), prev in zip(calls, ((0, 3), (3, 6), (6, 7)), (None, "scratch", "scratch")):
        assert dtype == torch.bfloat16 and torch.equal(got, refs[a:b].to(torch.bfloat16)) and scratch == prev
