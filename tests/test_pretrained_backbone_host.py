"""CPU: `pretrained_backbone` -- the ResNet body starts from torchvision's ImageNet file, as the reference's `pretrained=True`
does on its main process.  The checkpoints are synthetic files in torchvision's format (tests/imagenet_checkpoints.py) under a
temporary torch hub directory; nothing is downloaded."""
import hashlib
import os
import sys
import tempfile
import urllib.request

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import imagenet_checkpoints as ic
from monodetr_b200 import backbone as bb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ic.PREFIX


@pytest.fixture
def hub(tmp_path):
    """torch.hub.get_dir() -> an empty temporary directory, restored afterwards."""
    prev = torch.hub.get_dir()
    d = str(tmp_path / "hub")
    torch.hub.set_dir(d)
    try:
        yield d
    finally:
        torch.hub.set_dir(prev)


@pytest.fixture
def no_network(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("pretrained_backbone tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(urllib.request, "urlopen", refuse)


def _build(backbone, dilation, pretrained, seed=7):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    cfg = dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation)
    if pretrained is not None:
        cfg["pretrained_backbone"] = pretrained
    torch.manual_seed(seed)
    return build_monodetr(cfg)[0]


def _assert_loaded(model, plain, sd):
    """Body entries bit for bit from the file; every other entry and every requires_grad flag as in the random build."""
    state, ref = model.state_dict(), plain.state_dict()
    assert list(state) == list(ref)
    for k, v in state.items():
        if k.startswith(P):
            src = sd[k[len(P):]]
            assert v.dtype == torch.float32 and torch.equal(v.view(torch.int32), src.view(torch.int32)), k
        else:
            assert torch.equal(v, ref[k]), k
    assert [(n, p.requires_grad) for n, p in model.named_parameters()] == [(n, p.requires_grad) for n, p in plain.named_parameters()]


@pytest.mark.parametrize("dilation", [False, True])
@pytest.mark.parametrize("name", ic.NAMES)
def test_loads_the_hub_file_bit_for_bit(name, dilation, hub, no_network):
    sd = ic.synthetic_checkpoint(name, seed=len(name) + dilation)
    ic.write(sd, bb.imagenet_checkpoint_path(name))
    assert bb.imagenet_checkpoint_path(name) == os.path.join(hub, "checkpoints", bb.IMAGENET1K_V1[name][0])
    plain = _build(name, dilation, None)
    off = _build(name, dilation, False)
    assert all(torch.equal(a, b) for a, b in zip(plain.state_dict().values(), off.state_dict().values()))
    model = _build(name, dilation, True)
    assert len([k for k in model.state_dict() if k.startswith(P)]) == len(ic.body_spec(name, dilation))
    _assert_loaded(model, plain, sd)


def test_a_path_loads_the_same_way(tmp_path, hub, no_network):
    sd = ic.synthetic_checkpoint("resnet50", seed=3)
    path = ic.write(sd, str(tmp_path / "elsewhere" / "weights.pth"))
    _assert_loaded(_build("resnet50", False, path), _build("resnet50", False, False), sd)


def test_loading_draws_no_random_numbers(hub, no_network):
    ic.write(ic.synthetic_checkpoint("resnet50"), bb.imagenet_checkpoint_path("resnet50"))
    _build("resnet50", False, True)
    after_true = torch.rand(4)
    _build("resnet50", False, False)
    assert torch.equal(after_true, torch.rand(4))


def test_missing_file_raises_without_downloading(hub, no_network):
    path = bb.imagenet_checkpoint_path("resnext50_32x4d")
    with pytest.raises(FileNotFoundError) as e:
        _build("resnext50_32x4d", True, True)
    msg = str(e.value)
    assert path in msg and "'resnext50_32x4d'" in msg and "ResNeXt50_32X4D_Weights.IMAGENET1K_V1" in msg
    missing = os.path.join(hub, "nowhere.pth")
    with pytest.raises(FileNotFoundError, match="nowhere.pth"):
        _build("resnet50", False, missing)


def _bad(kind):
    sd = ic.synthetic_checkpoint("resnet50")
    if kind == "architecture":
        return ic.synthetic_checkpoint("resnet101"), "layer3.6"
    if kind == "missing":
        del sd["layer2.1.bn2.running_var"]
        return sd, "layer2.1.bn2.running_var"
    if kind == "extra":
        sd["layer4.0.conv2.bias"] = torch.zeros(512)
        return sd, "layer4.0.conv2.bias"
    if kind == "shape":
        return ic.synthetic_checkpoint("resnext50_32x4d"), "layer1.0.conv1.weight"
    if kind == "nan":
        sd["layer3.2.conv1.weight"][5, 7] = float("nan")
        return sd, "layer3.2.conv1.weight"
    if kind == "inf":
        sd["bn1.running_var"][3] = float("inf")
        return sd, "bn1.running_var"
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["architecture", "missing", "extra", "shape", "nan", "inf"])
def test_a_file_that_does_not_fit_raises(kind, hub, no_network):
    sd, offender = _bad(kind)
    ic.write(sd, bb.imagenet_checkpoint_path("resnet50"))
    with pytest.raises(ValueError, match=offender.replace(".", r"\.")):
        _build("resnet50", False, True)


def test_file_names_are_torchvisions():
    tv = pytest.importorskip("torchvision")
    for name, (fname, enum) in bb.IMAGENET1K_V1.items():
        url = getattr(tv.models, enum).IMAGENET1K_V1.url
        assert os.path.basename(url) == fname, name
    assert sorted(bb.IMAGENET1K_V1) == sorted(ic.NAMES)


# ---- world size 2: only rank 0 reads the file; the Trainer's broadcast brings it to rank 1 -------------------------------------
def _digest(t):
    """A tensor's bytes as a short string (the ranks report these instead of sending the tensors through the queue)."""
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def _worker(rank, world, store_path, q, workdir):
    os.environ["GLOO_SOCKET_IFNAME"] = "lo"
    dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, ROOT)
    import trainer_stubs as S
    from monodetr_b200 import trainer as T
    from monodetr_b200.optim import build_lr_scheduler
    torch.hub.set_dir(os.path.join(workdir, f"hub{rank}"))           # rank 1's hub directory stays empty
    os.chdir(os.path.join(workdir, str(rank)))
    reads = []
    load = torch.load
    torch.load = lambda *a, **k: (reads.append(a[0]), load(*a, **k))[1]
    try:
        model = _build("resnet50", False, True, seed=100 + rank)        # different random inits on the two ranks
    finally:
        torch.load = load
    before = {k: _digest(v) for k, v in model.state_dict().items() if k.startswith(P)}
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
    T.Trainer(dict(S.CFG, max_epoch=1), model, opt, [], None, sched, warm, S.ListLogger(), S.StubCriterion(), "stub")
    after = {k: _digest(v) for k, v in model.state_dict().items()}
    q.put((rank, reads, before, after))
    dist.barrier()
    dist.destroy_process_group()


def test_only_rank0_reads_and_the_trainer_broadcasts():
    tmp = tempfile.mkdtemp(prefix="mdb_gloo_pretrained_")
    for r in range(2):
        os.makedirs(os.path.join(tmp, str(r)))
    sd = ic.synthetic_checkpoint("resnet50", seed=11)
    path = ic.write(sd, os.path.join(tmp, "hub0", "checkpoints", bb.IMAGENET1K_V1["resnet50"][0]))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, os.path.join(tmp, "store"), q, tmp)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, reads0, before0, after0), (_, reads1, before1, after1) = res
    assert reads0 == [path] and reads1 == []
    for k, v in before0.items():
        assert v == _digest(sd[k[len(P):]]), k
    assert any(before1[k] != _digest(sd[k[len(P):]]) for k in before1)           # rank 1 built randomly
    assert list(after0) == list(after1)
    for k in after0:
        assert after0[k] == after1[k], k                                          # parameters and buffers
        if k.startswith(P):
            assert after1[k] == _digest(sd[k[len(P):]]), k
