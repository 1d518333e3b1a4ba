#!/usr/bin/env python
"""Multi-task balancing (Row MTL) at B = 65 536 on MMoE at the reference shape (d = 82, E = 3, H = 512, T = 3) and on PLE
at its defaults (one extraction network, 5 / 5 / 5 task experts, 10 shared, H = 256):

  * the training step (lookup, model body, loss, backward, balancing) with the plain sum, uncertainty weighting, GradNorm
    and PCGrad, median of --iters steps timed with CUDA events;
  * the loss kernel at T = 3 and B = 65 536 and 2^24, against its HBM floor (12*T*B bytes);
  * the Gram and PCGrad-combine kernels over the default shared parameters, against their HBM floors (T*P*4 and
    (T+1)*P*4 bytes at the data-sheet 3.35 TB/s) and against the torch equivalents (g.double() @ g.double().T, and the
    paper's vector-form loop), with the L2 flushed between timed calls.

Prints one JSON line per measurement, the first naming the GPU and its power limit.

    python tools/bench_multitask.py [--iters 20] [--batch 65536]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_layers import card, timeit  # noqa: E402
from recalgorithm_b200 import autograd, layers as L, multitask as MT, ops  # noqa: E402

HBM_GBS = 3350.0
NAMES = ("read_comment", "like", "click_avatar")


def build(kind, B):
    import model_bodies as M
    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    gen = torch.Generator(device="cuda").manual_seed(0)
    tables = autograd.EmbeddingTables([100000] * 10, 8, device="cuda")
    ids = torch.randint(-1, 100000, (B, 10), device="cuda", generator=gen)
    dense = torch.randn((B, 2), device="cuda", generator=gen)
    labels = {n: (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float() for n in NAMES}

    def forward():
        tables.grad_slices.clear()
        for v in store.vars.values():
            v.grad = None
        cat = autograd.lookup(tables, ids).reshape(B, -1)
        if kind == "mmoe":
            logits, _ = M.mmoe_logits(dense, cat, labels, task_names=NAMES, num_experts=3, expert_hidden_units=512)
        else:
            logits, _ = M.ple_logits(dense, cat, labels, task_names=NAMES)
        return logits, [labels[n] for n in NAMES]
    forward()
    return store, forward


def step_fns(kind, store, forward):
    shared = MT.mmoe_shared_parameters(store) if kind == "mmoe" else MT.ple_shared_parameters(store)
    uw = MT.UncertaintyWeighting(3)
    gn = MT.GradNorm(3, shared, lr=0.025)
    pc = MT.PCGrad(3, shared, seed=0)

    def plain():
        MT.multitask_sigmoid_ce(*forward(), "sum")[0].backward()

    def uncertainty():
        uw(*forward()).backward()

    def gradnorm():
        gn.loss(*forward()).backward(retain_graph=True)
        gn.update()

    def pcgrad():
        pc.backward(MT.multitask_sigmoid_ce(*forward(), "sum")[1])
    return shared, {"plain": plain, "uncertainty": uncertainty, "gradnorm": gradnorm, "pcgrad": pcgrad}


def torch_pcgrad(g, order):
    out = torch.zeros_like(g[0])
    for i in range(g.shape[0]):
        gi = g[i].clone()
        for j in order:
            if j == i:
                continue
            dot = gi @ g[j]
            gi -= torch.where(dot < 0, dot / (g[j] @ g[j]), torch.zeros_like(dot)) * g[j]
        out += gi
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=65536)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    no_flush = torch.empty(0, dtype=torch.uint8, device="cuda")
    for kind in ("mmoe", "ple"):
        store, forward = build(kind, args.batch)
        shared, fns = step_fns(kind, store, forward)
        T, P = 3, sum(p.numel() for p in shared)
        for name, fn in fns.items():
            m, best = timeit(fn, args.iters, no_flush)
            print(json.dumps({"model": kind, "B": args.batch, "step": name, "ms_median": m, "ms_best": best}), flush=True)
        g = torch.randn((T, P), device="cuda")
        gram = ops.multitask_gram(g)
        order = torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda")
        rows = [("ctr_multitask_gram", lambda: ops.multitask_gram(g), T * P * 4),
                ("torch_gram_float64", lambda: g.double() @ g.double().T, T * P * 4),
                ("ctr_pcgrad_combine", lambda: ops.pcgrad_combine(g, gram, order), (T + 1) * P * 4),
                ("torch_pcgrad_vector_form", lambda: torch_pcgrad(g, [2, 0, 1]), (T + 1) * P * 4)]
        for name, fn, nbytes in rows:
            m, best = timeit(fn, args.iters, flush)
            floor_us = nbytes / (HBM_GBS * 1e9) * 1e6
            print(json.dumps({"model": kind, "kernel": name, "T": T, "P": P, "us_median": m * 1e3, "us_best": best * 1e3,
                              "hbm_floor_us": floor_us, "bytes": nbytes, "l2": "flushed between iterations"}), flush=True)
        if kind == "mmoe":                                      # the loss kernel's one cluster, at two batch sizes
            for B in (args.batch, 1 << 24):
                x = torch.randn((T, B), device="cuda")
                z = (torch.rand((T, B), device="cuda") < 0.3).float()
                m, best = timeit(lambda: ops.multitask_sigmoid_ce(x, z, 0), args.iters, flush)
                nbytes = 12 * T * B
                print(json.dumps({"kernel": "ctr_multitask_sigmoid_ce", "T": T, "B": B, "us_median": m * 1e3,
                                  "us_best": best * 1e3, "hbm_floor_us": nbytes / (HBM_GBS * 1e9) * 1e6, "bytes": nbytes,
                                  "l2": "flushed between iterations"}), flush=True)
                del x, z
        del store, forward, fns, shared
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
