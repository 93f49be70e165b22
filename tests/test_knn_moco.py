"""CPU: the kNN memory, the contrastive loss and the bank-scan entry points of csrc/pv_bank.cu - argument errors, the
k / dim caps, host-side KnnMemory behaviour against the reference's, and a launch-name ledger: every launch site and
entry point of pv_bank.cu has a GPU test in tests/test_gpu_knn_moco.py that asserts it ran."""
import math
import os
import re
import types

import pytest
import torch

from pytorchvideo_b200 import contrastive as K
from pytorchvideo_b200.losses import ContrastiveLoss
from pytorchvideo_b200.models.knn_memory import KnnMemory

TESTS = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(TESTS), "pytorchvideo_b200", "csrc")


def test_knn_memory_draw_and_buffers_match_reference():
    """The reference draws torch.rand(length, dim).mul_(2 stdv).add_(-stdv) on the device; memory is a buffer."""
    torch.manual_seed(4)
    knn = KnnMemory(50, 12, momentum=0.5, downstream_classes=7, temperature=0.1, knn_k=3)
    torch.manual_seed(4)
    stdv = 1.0 / math.sqrt(12 / 3)
    assert torch.equal(knn.memory, torch.rand(50, 12).mul_(2 * stdv).add_(-stdv))
    assert list(knn.state_dict()) == ["memory"]
    assert (knn.length, knn.dim, knn.momentum, knn.downstream_classes, knn.temperature, knn.knn_k) == (
        50, 12, 0.5, 7, 0.1, 3)
    ind = torch.tensor([[3], [7]])
    assert torch.equal(knn.get(ind), knn.memory[[3, 7]].view(2, -1, 12))


def test_init_knn_labels_reads_the_dataset_and_resizes():
    videos = [("v%d" % i, {"label": (3 * i) % 5}) for i in range(9)]
    loader = types.SimpleNamespace(dataset=types.SimpleNamespace(_labeled_videos=videos))
    knn = KnnMemory(4, 6)
    knn.init_knn_labels(loader)
    assert knn.num_imgs == 9 and knn.length == 9 and tuple(knn.memory.shape) == (9, 6)
    assert knn.train_labels.dtype == torch.int64 and knn.train_labels.tolist() == [(3 * i) % 5 for i in range(9)]
    assert "memory" not in dict(knn.named_buffers())       # the reference's resize rebinds it as a plain attribute


def test_eval_knn_before_labels_and_cpu_tensors_raise():
    knn = KnnMemory(10, 4, knn_k=2)
    with pytest.raises(AttributeError):
        knn.eval_knn(torch.zeros(2, 4))
    knn.train_labels = torch.zeros(10, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="GPU"):
        knn.eval_knn(torch.zeros(2, 4))
    with pytest.raises(RuntimeError, match="GPU"):
        knn.update(torch.zeros(2, 4), torch.tensor([0, 1]))
    assert knn(torch.zeros(1)) is None


def test_caps_and_argument_errors():
    q = torch.zeros(2, 8)
    with pytest.raises(NotImplementedError):
        K.bank_topk(q, torch.zeros(2000, 8), 1025, torch.zeros(2000, dtype=torch.int64), 3, 0.1)
    with pytest.raises(NotImplementedError):
        K.bank_topk(torch.zeros(2, 2049), torch.zeros(10, 2049), 1, torch.zeros(10, dtype=torch.int64), 3, 0.1)
    with pytest.raises(RuntimeError):                    # no CPU path
        K.bank_topk(q, torch.zeros(10, 8), 2, torch.zeros(10, dtype=torch.int64), 3, 0.1)
    with pytest.raises(RuntimeError):
        K.bank_update(torch.zeros(10, 8), q, torch.tensor([0, 1]), 0.5)
    with pytest.raises(NotImplementedError):
        K.queue_ce(q, torch.zeros(4, 8), torch.zeros(2, 2, 8), 0.1, reduction="sum")
    with pytest.raises(NotImplementedError):
        ContrastiveLoss(reduction="sum")
    loss = ContrastiveLoss()
    assert loss.reduction == "mean" and loss.temperature == 0.1
    with pytest.raises(RuntimeError):
        loss(torch.zeros(3, 5))
    with pytest.raises(RuntimeError):
        loss(torch.zeros(3, 5, requires_grad=True))


def test_distributed_update_is_refused(monkeypatch):
    knn = KnnMemory(10, 4)
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda *a: 2)
    with pytest.raises(NotImplementedError):
        knn.update(torch.zeros(2, 4), torch.tensor([0, 1]))


# ---- launch-name ledger of pv_bank.cu --------------------------------------------------------------------------------
# entry point -> the GPU tests that call it; launch name -> the GPU tests that assert it ran
ENTRY_TESTS = {
    "pv_bank_topk": ["test_bank_topk_vs_f64", "test_bank_topk_k400_configuration"],
    "pv_bank_update": ["test_bank_update_bit_exact", "test_bank_update_out_of_range_writes_nothing"],
    "pv_queue_ce": ["test_queue_ce_vs_f64", "test_contrastive_loss_vs_f64"],
}
ENTRY_NOT_CALLED = {"pv_bank_workspace": "host only: the workspace size, called by every bank_topk / queue_ce"}


def bank_source():
    return open(os.path.join(CSRC, "pv_bank.cu")).read()


def gpu_tests():
    return "".join(open(os.path.join(TESTS, f)).read() for f in ("test_gpu_knn_moco.py", "test_gpu_moco_golden.py"))


def launch_names(src):
    return set(re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', src)) | set(re.findall(r'PV_TOPK\(\d, \w+, "([^"]+)"\)', src))


def asserted_names(tests):
    """Launch names the GPU tests spell out as string literals (a test asserts each with _ran or by comparing)."""
    return set(re.findall(r'"(\w+_kernel(?:<[^"%]*>)?)"', tests))


def ledger_problems(src, tests, entry_tests):
    out = ["launch name %s: no GPU test asserts it" % n for n in sorted(launch_names(src) - asserted_names(tests))]
    entries = set(re.findall(r'extern "C" int (pv_\w+)\(', src))
    out += ["entry point %s: no GPU test calls it" % e for e in sorted(entries - set(entry_tests) - set(ENTRY_NOT_CALLED))]
    for e, names in sorted(entry_tests.items()):
        out += ["%s: GPU test %s is missing" % (e, n) for n in names if "def %s(" % n not in tests]
    return out


def test_ledger_covers_every_launch_site_and_entry_point():
    src = bank_source()
    assert len(launch_names(src)) == 11, sorted(launch_names(src))
    assert not ledger_problems(src, gpu_tests(), ENTRY_TESTS), ledger_problems(src, gpu_tests(), ENTRY_TESTS)


def test_ledger_fails_on_a_new_launch_site_or_a_lost_test():
    src, tests = bank_source(), gpu_tests()
    assert ledger_problems(src + '\nvoid f() { PV_LAUNCH_OK("new_kernel"); }\n', tests, ENTRY_TESTS)
    assert ledger_problems(src + '\nextern "C" int pv_new_entry(void* stream) { return 0; }\n', tests, ENTRY_TESTS)
    assert ledger_problems(src, tests.replace("def test_queue_ce_vs_f64(", "def renamed("), ENTRY_TESTS)
    assert ledger_problems(src, tests.replace('"bank_update_kernel"', '"other"'), ENTRY_TESTS)
    assert ledger_problems(src, tests.replace('"bank_score_kernel<lse,32,scalar>"', '"other"'), ENTRY_TESTS)
    assert ledger_problems(src, tests.replace('"bank_score_kernel<topk,8,scalar>"', '"other"'), ENTRY_TESTS)


# ---- MoCo v2 and the kNN memory against tests/golden/knn_moco.pt (the trainer's own modules, on the CPU) ----------
GOLD = os.path.join(TESTS, "golden", "knn_moco.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.mark.parametrize("name", ["moco_linear_v2", "moco_linear_v3", "moco_slow_r50"])
def test_moco_tree_state_dict_and_queue_draw_match_reference(gold, name):
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.models.moco_v2 import MOCO, MoCoQueue, create_mlp_util, create_moco_resnet_50
    from pytorchvideo_b200.models.resnet import create_resnet
    ns = types.SimpleNamespace(MOCO=MOCO, create_moco_resnet_50=create_moco_resnet_50, create_mlp_util=create_mlp_util,
                               create_resnet=create_resnet)
    g = gold["moco"][name]
    model, views, k, dim = TS.build_moco_case(name, ns)
    assert TS.tree_digests(model) == g["tree"]
    torch.manual_seed(TS.MOCO_QUEUE_SEED)
    queue = MoCoQueue(dim, k)
    ref_keys = [n for n in g["module_keys"] if not n.startswith(("model.", "knn_memory."))]
    assert list(queue.state_dict()) == ref_keys == ["ptr", "queue_x"]
    if isinstance(g["queue0"], torch.Tensor):
        assert torch.equal(queue.queue_x, g["queue0"])
    else:
        assert TS.tensor_checksum(queue.queue_x) == g["queue0"]
    with pytest.raises(RuntimeError):                    # eval-mode engine, no CPU path
        model(views[0])


def test_create_mlp_util_matches_reference(gold):
    from pytorchvideo_b200.models.moco_v2 import create_mlp_util
    assert repr(create_mlp_util(12, 8, 32, 3, norm=torch.nn.BatchNorm1d)) == gold["mlp"]["repr"]
    assert [getattr(m, "xavier_init", None) for m in create_mlp_util(12, 8, 32, 3, norm=None)] == gold["mlp"]["xavier"]


@pytest.mark.parametrize("name", ["m1000_d8_k1", "k400_n64"])
def test_knn_memory_tree_matches_reference(gold, name):
    from pytorchvideo_b200 import testing as TS
    knn, _ = TS.knn_case(name, KnnMemory)
    assert TS.tree_digests(knn) == gold["knn"][name]["tree"]


def test_moco_refuses_distributed(monkeypatch):
    from pytorchvideo_b200.models.moco_v2 import MoCoQueue
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda *a: 2)
    with pytest.raises(NotImplementedError):
        MoCoQueue(8, 16).compute_keys(None, [torch.zeros(4, 16)])
