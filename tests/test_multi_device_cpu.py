"""Host logic of in-process sharding (no GPU): VRGDG_DEVICES parsing against faked device queries, and the shard plan."""
import importlib

import pytest
import torch


@pytest.fixture
def rt(pkg):
    return importlib.import_module(pkg.__name__ + "._runtime")


@pytest.fixture
def fake_cards(monkeypatch):
    """Four visible cards: cuda:1 is compute capability 8.0, the others 9.0."""
    caps = [(9, 0), (8, 0), (9, 0), (9, 0)]

    def cap(i):
        assert 0 <= i < len(caps), "queried a device that is not visible"
        return caps[i]
    monkeypatch.setattr(torch.cuda, "device_count", lambda: len(caps))
    monkeypatch.setattr(torch.cuda, "get_device_capability", cap)
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda i: "A100-SXM4-80GB" if caps[i] == (8, 0) else "H100 80GB HBM3")
    return caps


def _idx(devs):
    return [d.index for d in devs] if devs is not None else None


@pytest.mark.parametrize("value", [None, "", "  "])
def test_unset_or_empty_means_one_compute_device(rt, fake_cards, monkeypatch, value):
    if value is None:
        monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    else:
        monkeypatch.setenv("VRGDG_DEVICES", value)
    assert rt.devices_from_env() is None


@pytest.mark.parametrize("value, want", [("all", [0, 2, 3]), ("ALL", [0, 2, 3]), ("0", [0]), ("3,0", [3, 0]), (" 2 , 3 ", [2, 3])])
def test_accepted_values(rt, fake_cards, monkeypatch, value, want):
    monkeypatch.setenv("VRGDG_DEVICES", value)
    devs = rt.devices_from_env()
    assert _idx(devs) == want and all(d.type == "cuda" for d in devs)


@pytest.mark.parametrize("value, names", [
    ("0,0", "cuda:0"),                 # duplicate
    ("2,3,2", "cuda:2"),               # duplicate
    ("4", "cuda:4"),                   # not visible
    ("-1", "cuda:-1"),                 # not visible
    ("1", "cuda:1 (A100-SXM4-80GB)"),  # compute capability 8.0
    ("0,x", "'x'"),
    ("0,,2", "''"),
    ("cuda:0", "'cuda:0'"),
])
def test_rejected_values_name_the_device(rt, fake_cards, monkeypatch, value, names):
    monkeypatch.setenv("VRGDG_DEVICES", value)
    with pytest.raises(ValueError) as e:
        rt.devices_from_env()
    assert names in str(e.value)


def test_all_without_a_9_0_device_is_an_error(rt, monkeypatch):
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 2)
    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda i: (8, 6))
    monkeypatch.setenv("VRGDG_DEVICES", "all")
    with pytest.raises(ValueError, match="compute capability 9.0"):
        rt.devices_from_env()


def test_shard_plan_is_contiguous_and_covering(rt):
    for n in range(0, 13):
        for k in range(1, 6):
            plan = rt.shard_plan(n, k)
            assert len(plan) == k
            start = 0
            for a, b in plan:
                assert a == start and b >= a         # each shard starts where the previous one stopped: its absolute first frame
                start = b
            assert start == n
            sizes = [b - a for a, b in plan]
            assert sizes == sorted(sizes, reverse=True) and sizes[0] - sizes[-1] <= 1   # the first shards take the remainder
    assert rt.shard_plan(7, 3) == [(0, 3), (3, 5), (5, 7)]
    assert rt.shard_plan(1, 2) == [(0, 1), (1, 1)]                                     # fewer frames than devices: an empty shard


def test_device_lists_must_name_cuda_devices(pkg, rt):
    for bad in ([], ["cpu"], ["cuda:0", "cpu"]):
        with pytest.raises(ValueError):
            pkg.chain.PostChain(devices=bad)
        with pytest.raises(ValueError):
            rt.stream_frames_sharded(torch.zeros(2, 4, 4, 3), lambda d: None, 1, "cpu", bad)
