"""``bench.py --driver vae | vae_cl | cpc`` — benchmark configuration 5 (VAE + CPC encoders, K = N workers, one per GPU).

Same contract as the headline arm (``bench.py:run_ours``): one engine per process, W + prime warm-up steps, EXACTLY K
timed optimizer steps per worker bracketed by barrier + synchronize, placed so that they straddle the first
aggregation of the schedule (so the fused NVLink aggregation of the active layer is inside the number), CUDA events,
max over ranks.  A *step* is one ``optimizer.step(closure)`` on every worker: Adam for the VAE (graph-replayed), the
stochastic L-BFGS of the reference (4 backward + 12-16 forward passes per step at ``max_iter=4``) for VAE-CL / CPC.
``value`` = images/s (CPC: baselines/s, each baseline = 9 patches of 8 x 32 x 32) of the whole job.

Reference drivers: /root/reference/src/federated_vae.py, federated_vae_cl.py, federated_cpc.py.
"""
from __future__ import annotations

import os
import time

import torch


def run_aux_bench(args) -> dict:
    from bench import PRIME_STEPS, ClockSampler, _max_over_ranks, straddle_window
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.algo.strategies import FedAvg
    from federated_pytorch_test_b200.api import common, federated_cpc, federated_vae, federated_vae_cl
    from federated_pytorch_test_b200.ops import cuda_ops

    N, K, W = args.gpus, args.steps, args.warmup
    world = int(os.environ.get("WORLD_SIZE", "1"))
    assert world == N or (N == 1 and world == 1), "launch with torchrun --nproc-per-node N for N > 1"
    if args.driver == "cpc":
        per_round, batch = 10, 128                       # Niter = 10 minibatches per worker per round (federated_cpc.py:34)
        mod, task_cls = federated_cpc, federated_cpc.CPCTask
        first = straddle_window(K, W, 1, per_round)
        rounds = -(-(first + K) // per_round) + 1
        cfg = mod.Config(K=N, Nloop=1000, Nadmm=rounds, Niter=per_round, load_model=False, init_model=True, save_model=False,
                         be_verbose=False, check_results=False, graphs=not args.no_graphs, fast=not args.no_fast, collective=args.collective, seed=69)
    else:
        per_round, batch = 49, 128                       # the K = 8 shard: 49 minibatches per round
        mod = federated_vae if args.driver == "vae" else federated_vae_cl
        task_cls = federated_vae.VAETask if args.driver == "vae" else federated_vae_cl.VAECLTask
        first = straddle_window(K, W, PRIME_STEPS, per_round)
        b_host = -(-(first + K) // per_round) * per_round           # first step served from pinned host memory (e2e window)
        first_e = straddle_window(K, W, b_host, b_host + per_round)
        rounds = -(-(first_e + K) // per_round) + 1 if not args.no_e2e else -(-(first + K) // per_round) + 1
        kw = dict(K=N, Nloop=1000, Nadmm=rounds, Nepoch=1, check_results=False, save_model=False, be_verbose=False,
                  graphs=not args.no_graphs, fast=not args.no_fast, collective=args.collective, max_minibatches=per_round, seed=69)
        cfg = mod.Config(**kw)
    last = first + K
    e2e_on = args.driver != "cpc" and not args.no_e2e          # CPC draws synthetic LOFAR baselines on the device: no host path
    if not e2e_on:
        first_e = -1
    last_e = first_e + K
    topo, coll = common.setup_runtime(cfg)
    task = task_cls(cfg, topo)
    ecfg = common.engine_config(cfg, Nepoch=1, diagnostics="pre") if args.driver == "cpc" else common.engine_config(cfg)
    eng = Engine(task, topo, FedAvg(coll, topo), coll, ecfg, log=lambda m: None)
    dev = topo.device
    ev = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]
    st = {}
    sampler = ClockSampler(dev.index or 0) if topo.is_root else None
    if sampler:
        sampler.start()          # early: NVML start-up stalls launches on every GPU of the box (see bench.py)

    ev_e = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]
    slots = [torch.zeros((), dtype=torch.float32).pin_memory() for _ in range(2)] if dev.type == "cuda" else None
    slot_ev = [torch.cuda.Event(), torch.cuda.Event()]
    pending = []

    def to_host_loaders():
        from federated_pytorch_test_b200.data.cifar import CifarData

        d = task.data
        task.data = CifarData(d.train_images.cpu(), d.train_labels.cpu(), d.test_images.cpu(), d.test_labels.cpu()).to(dev, pin=True)
        task._loaders.clear()

    def hook(e: Engine):
        n = e.steps_done
        if e2e_on and first_e <= n - 1 < last_e and e.last_loss1 is not None:      # the step just finished was an e2e step
            i = n & 1
            slots[i].copy_(e.last_loss1.detach().reshape(()), non_blocking=True)     # D2H of this step's result
            slot_ev[i].record()
            pending.append(i)
            while len(pending) > (0 if n >= last_e else 1):                          # read the previous step's value
                j = pending.pop(0)
                slot_ev[j].synchronize()
                st["loss"] = float(slots[j])
        if e2e_on and n == first_e:
            topo.barrier()
            torch.cuda.synchronize(dev)
            st.update(te0=time.perf_counter(), ae0=e.aggregations_done)
            ev_e[0].record()
        elif e2e_on and n == last_e:
            ev_e[1].record()
            torch.cuda.synchronize(dev)
            topo.barrier()
            st.update(te1=time.perf_counter(), aggs_e=e.aggregations_done - st["ae0"])
            e.stop_requested = True
        if n == first:
            topo.barrier()
            torch.cuda.synchronize(dev)
            st["smi0"] = sampler.mark() if sampler else 0
            st.update(l0=cuda_ops.launch_count(), g0=e.graph_kernel_launches, a0=e.aggregations_done, t0=time.perf_counter())
            ev[0].record()
        elif n == last:
            ev[1].record()
            torch.cuda.synchronize(dev)
            topo.barrier()
            st.update(t1=time.perf_counter(), launches=(cuda_ops.launch_count() - st["l0"]) + (e.graph_kernel_launches - st["g0"]),
                      aggs=e.aggregations_done - st["a0"], clocks=sampler.window(st["smi0"], sampler.mark()) if sampler else None)
            if e2e_on:
                to_host_loaders()          # from the next round on: pinned host memory -> native batch assembler -> async H2D
            else:
                e.stop_requested = True

    eng.step_hook = hook
    eng.run()
    if sampler:
        sampler.stop()
    ms = _max_over_ranks(ev[0].elapsed_time(ev[1]), dev)
    wall = _max_over_ranks((st["t1"] - st["t0"]) * 1e3, dev)
    out = {
        "metric": "train_images_per_sec", "value": batch * N * K / (ms / 1e3), "unit": "images/s" if args.driver != "cpc" else "baselines/s",
        "n_gpus": N, "steps": K, "warmup": W, "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "tf32 conv / fp32 dense", "data": "synthetic", "impl": "ours",
        "config": {"model": {"vae": "AutoEncoderCNN", "vae_cl": "AutoEncoderCNNCL(K=10,L=32)", "cpc": "EncoderCNN/ContextgenCNN/PredictorCNN(L=256,R=32)"}[args.driver],
                   "algo": "fedavg", "optimizer": "adam" if args.driver == "vae" else "LBFGSNew (stochastic)", "global_batch": batch * N, "K": N,
                   "parallelism": "fed%d (one replica per GPU, layer-wise FedAvg over NVLink)" % N, "steps_per_round": per_round,
                   "timed_steps": [first, last], "aggregations_in_window": st.get("aggs"), "collective": coll.name,
                   "cuda_graphs": bool(cfg.graphs), "wall_ms_per_step": wall / K,
                   "timing": "CUDA events, barrier+synchronize both sides, max over ranks"},
        "clocks": st.get("clocks"), "gpu_launches": st.get("launches"),
        "e2e": {"unavailable": "the CPC driver draws its synthetic LOFAR baselines on the device (the reference reads h5 files that do not exist here)"},
    }
    if e2e_on:
        ms_e = _max_over_ranks(ev_e[0].elapsed_time(ev_e[1]), dev)
        loader = task.loader(topo.local_workers[0])
        out["e2e"] = {"value": batch * N * K / (ms_e / 1e3), "unit": out["unit"], "ms_per_step": ms_e / K,
                      "wall_ms_per_step": _max_over_ranks((st["te1"] - st["te0"]) * 1e3, dev) / K,
                      "h2d_bytes_per_step": loader.h2d_bytes_per_batch * (1 if loader.host_resident else 0), "d2h_bytes_per_step": 4,
                      "timed_steps": [first_e, last_e], "aggregations_in_window": st.get("aggs_e"), "last_loss_read_by_host": st.get("loss"),
                      "note": "same engine, dataset moved to pinned host memory after the device window: native batch assembler, async H2D of "
                              "every uint8 batch, every step's loss copied D2H into pinned memory and read by the host one step later"}
    return out if topo.is_root else {}
