"""Times the bank scans of csrc/pv_bank.cu on the GPU against the reference's eager torch expressions on the same card,
the two arms alternated: KnnMemory.eval_knn at the trainer's kinetics_k400 configuration (239,975 rows, dim 128,
k = 200, 400 classes), KnnMemory.update, MoCo's queue cross entropy at K = 65,536, and a Slow-R50 MoCo step
(batch 8, 8 x 224^2, two views, K = 65,536).  The fused eval_knn and update calls read their device error flag, one
device-to-host synchronise per call, which the eager arm does not make.  Bytes and FLOPs are computed
from the shapes.  Prints the card's name, power limit and max SM clock first.

    python tools/bench_knn_moco.py [--iters 50]
"""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import contrastive as K  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:              # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters             # us


def compare(name, fused, eager, nbytes, flops, iters, rounds=5):
    for f in (fused, eager):
        f()
    torch.cuda.synchronize()
    tf, te = [], []
    for _ in range(rounds):
        tf.append(timed(fused, iters))
        te.append(timed(eager, iters))
    f, e = min(tf), min(te)
    print("%-38s fused %9.1f us  eager %9.1f us  x%.2f  | %7.1f MB %6.2f GFLOP -> fused %6.0f GB/s %5.1f TFLOP/s" % (
        name, f, e, e / f, nbytes / 1e6, flops / 1e9, nbytes / f / 1e3, flops / f / 1e6))


def eager_knn(q, memory, labels, k, C, T):
    dist = torch.einsum("nc,mc->nm", q, memory)
    yd, yi = dist.topk(k, dim=1, largest=True, sorted=True)
    retrieval = torch.gather(labels.view(1, -1).expand(q.shape[0], -1), 1, yi)
    onehot = torch.zeros((q.shape[0] * k, C), device=q.device).scatter_(1, retrieval.view(-1, 1), 1)
    w = yd.clone().div_(T).exp_()
    return torch.sum(onehot.view(q.shape[0], -1, C) * w.view(q.shape[0], -1, 1), 1)


def eager_update(memory, mem, ind, m):
    old = memory[ind].view(mem.shape[0], 1, -1)
    upd = F.normalize(mem.view(mem.shape[0], 1, -1) * m + old * (1 - m), p=2, dim=1)
    memory[ind, :] = upd.squeeze()


def eager_queue(q, queue, key, T):
    neg = torch.einsum("nc,kc->nk", q, queue)
    pos = torch.einsum("nc,nc->n", q, key).unsqueeze(-1)
    lg = torch.div(torch.cat([pos, neg], 1), T)
    return F.cross_entropy(lg, torch.zeros(q.shape[0], dtype=torch.long, device=q.device))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    print("card:", card())
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    M, dim, k, C, T = 239975, 128, 200, 400, 0.1
    memory = F.normalize(torch.randn((M, dim), device=dev, generator=g), dim=1)
    labels = torch.randint(0, C, (M,), device=dev, generator=g)
    for N in (64, 256):
        q = F.normalize(torch.randn((N, dim), device=dev, generator=g), dim=1)
        _, _, p = K.bank_topk(q, memory, k, labels, C, T)
        ref = eager_knn(q, memory, labels, k, C, T)
        print("  eval_knn N=%d max |fused - eager| / max|eager| = %.2e" % (
            N, float((p - ref).abs().max() / ref.abs().max())))
        compare("eval_knn K400 N=%d" % N, lambda: K.bank_topk(q, memory, k, labels, C, T),
                lambda: eager_knn(q, memory, labels, k, C, T), M * dim * 4 * ((N + 31) // 32), 2.0 * N * M * dim, a.iters)
    N = 64
    mem = torch.randn((N, dim), device=dev, generator=g)
    ind = torch.randperm(M, device=dev, generator=g)[:N]
    bank_a, bank_b = memory.clone(), memory.clone()
    compare("update N=64", lambda: K.bank_update(bank_a, mem, ind, 0.5), lambda: eager_update(bank_b, mem, ind, 0.5),
            N * dim * 4 * 3, N * dim * 5.0, a.iters)
    Kq = 65536
    queue = F.normalize(torch.randn((Kq, dim), device=dev, generator=g), dim=1)
    for N in (8, 32):
        q = F.normalize(torch.randn((N, dim), device=dev, generator=g), dim=1)
        keys = F.normalize(torch.randn((2, N, dim), device=dev, generator=g), dim=2)
        got = K.queue_ce(q, queue, keys, 0.2, 0)
        ref = eager_queue(q, queue, keys[1], 0.2)
        print("  queue_ce N=%d |fused - eager| = %.2e (loss %.4f)" % (N, abs(float(got) - float(ref)), float(ref)))
        compare("queue_ce K=65536 N=%d V=2" % N, lambda: K.queue_ce(q, queue, keys, 0.2, 0),
                lambda: eager_queue(q, queue, keys[1], 0.2), Kq * dim * 4, 2.0 * N * Kq * dim, a.iters)
    moco_step(10)


def moco_step(iters):
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.losses import ContrastiveLoss
    from pytorchvideo_b200.models.moco_v2 import MoCoQueue, create_moco_resnet_50
    torch.manual_seed(0)
    model = TS.randomize_model(create_moco_resnet_50(), seed=1).eval().to("cuda")
    queue = MoCoQueue(128, 65536).to("cuda")
    views = [torch.rand((8, 3, 8, 224, 224), device="cuda") for _ in range(2)]
    loss = ContrastiveLoss()
    for _ in range(3):
        queue.step(model, views, loss)
    torch.cuda.synchronize()
    t = timed(lambda: queue.step(model, views, loss), iters)
    print("%-38s fused %9.1f us  (momentum update + refresh, 2 key and 2 online Slow-R50 passes, 2 queue CEs)" % (
        "MoCo Slow-R50 step, batch 8, V=2", t))


if __name__ == "__main__":
    main()
