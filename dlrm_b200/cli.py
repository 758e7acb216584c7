"""`python dlrm_s_pytorch.py <flags>` -- the reference's command line (dlrm_s_pytorch.py:902-1021) driving
the H100 engine, so that `bench/dlrm_s_benchmark.sh` runs unmodified from this repo's root.

Every flag of the reference is accepted with the same default.  Flags that select subsystems outside
the hot path (datasets, QR/MD embeddings, quantisation, ONNX, mlperf logging, ...) exit with the
reference's style of error.  --test-freq / --inference-only run the reference's test pass (inference(),
:759-900), --save-model / --load-model write and read the reference's checkpoint dictionary (:860-866,
:1399-1456, :1703-1715; a checkpoint written by the reference loads here and vice versa), --enable-profiling
and --debug-mode do what they do there.  --max-ind-range and --mlperf-grad-accum-iter only act on the
dataset / mlperf-logging paths in the reference (rejected above), so they have no effect here either.  The random-data generator draws from numpy's global RNG in EXACTLY the
reference's order (dlrm_data_pytorch.py:899-960 and :838-846; re-seeded at batch 0 of every epoch,
:637-638), and parameters are initialised in the reference's order, so for the same
`--numpy-rand-seed` the inputs and initial weights are bit-identical to the reference's and the printed
loss curve can be compared directly (tests/test_gpu_facade.py does so against a recorded reference run).
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np
import torch


def dash_separated_ints(value):
    for val in value.split("-"):
        try:
            int(val)
        except ValueError:
            raise argparse.ArgumentTypeError("%s is not a valid dash separated list of ints" % value)
    return value


def dash_separated_floats(value):
    for val in value.split("-"):
        try:
            float(val)
        except ValueError:
            raise argparse.ArgumentTypeError("%s is not a valid dash separated list of floats" % value)
    return value


# (flag, type-or-action, default) in the reference's order, dlrm_s_pytorch.py:908-1021
_FLAGS = [
    ("--arch-sparse-feature-size", int, 2), ("--arch-embedding-size", dash_separated_ints, "4-3-2"),
    ("--arch-mlp-bot", dash_separated_ints, "4-3-2"), ("--arch-mlp-top", dash_separated_ints, "4-2-1"),
    ("--arch-interaction-itself", "store_true", False), ("--weighted-pooling", str, None),
    ("--md-flag", "store_true", False), ("--md-threshold", int, 200), ("--md-temperature", float, 0.3),
    ("--md-round-dims", "store_true", False), ("--qr-flag", "store_true", False), ("--qr-threshold", int, 200),
    ("--qr-operation", str, "mult"), ("--qr-collisions", int, 4), ("--activation-function", str, "relu"),
    ("--loss-function", str, "mse"), ("--loss-weights", dash_separated_floats, "1.0-1.0"),
    ("--loss-threshold", float, 0.0), ("--round-targets", bool, False), ("--data-size", int, 1),
    ("--num-batches", int, 0), ("--rand-data-dist", str, "uniform"), ("--rand-data-min", float, 0),
    ("--rand-data-max", float, 1), ("--rand-data-mu", float, -1), ("--rand-data-sigma", float, 1),
    ("--data-trace-file", str, "./input/dist_emb_j.log"), ("--data-set", str, "kaggle"),
    ("--raw-data-file", str, ""), ("--processed-data-file", str, ""), ("--data-randomize", str, "total"),
    ("--data-trace-enable-padding", bool, False), ("--max-ind-range", int, -1),
    ("--data-sub-sample-rate", float, 0.0), ("--num-indices-per-lookup", int, 10),
    ("--num-indices-per-lookup-fixed", bool, False), ("--num-workers", int, 0),
    ("--memory-map", "store_true", False), ("--mini-batch-size", int, 1), ("--nepochs", int, 1),
    ("--learning-rate", float, 0.01), ("--print-precision", int, 5), ("--numpy-rand-seed", int, 123),
    ("--sync-dense-params", bool, True), ("--optimizer", str, "sgd"),
    ("--dataset-multiprocessing", "store_true", False), ("--inference-only", "store_true", False),
    ("--quantize-mlp-with-bit", int, 32), ("--quantize-emb-with-bit", int, 32), ("--save-onnx", "store_true", False),
    ("--use-gpu", "store_true", False), ("--local_rank", int, -1), ("--dist-backend", str, ""),
    ("--print-freq", int, 1), ("--test-freq", int, -1), ("--test-mini-batch-size", int, -1),
    ("--test-num-workers", int, -1), ("--print-time", "store_true", False),
    ("--print-wall-time", "store_true", False), ("--debug-mode", "store_true", False),
    ("--enable-profiling", "store_true", False), ("--plot-compute-graph", "store_true", False),
    ("--tensor-board-filename", str, "run_kaggle_pt"), ("--save-model", str, ""), ("--load-model", str, ""),
    ("--mlperf-logging", "store_true", False), ("--mlperf-acc-threshold", float, 0.0),
    ("--mlperf-auc-threshold", float, 0.0), ("--mlperf-bin-loader", "store_true", False),
    ("--mlperf-bin-shuffle", "store_true", False), ("--mlperf-grad-accum-iter", int, 1),
    ("--lr-num-warmup-steps", int, 0), ("--lr-decay-start-step", int, 0), ("--lr-num-decay-steps", int, 0),
]


def build_parser():
    p = argparse.ArgumentParser(description="Train Deep Learning Recommendation Model (DLRM) -- dlrm_b200")
    for name, typ, default in _FLAGS:
        if typ == "store_true":
            p.add_argument(name, action="store_true", default=default)
        else:
            p.add_argument(name, type=typ, default=default)
    p.add_argument("--arch-interaction-op", type=str, choices=["dot", "cat"], default="dot")
    # the reference's choices (:941-945) plus "synthetic": its RandomDataset implements the trace-driven
    # generator but its parser cannot select it
    p.add_argument("--data-generation", type=str, choices=["random", "dataset", "internal", "synthetic"],
                   default="random")
    # dlrm_b200 addition (not in the reference): GEMM back end
    p.add_argument("--gemm", type=str, default="tc", choices=["tc", "tc_bf16", "simt"])
    return p


def reference_order_batch(m_den, ln_emb, n, num_indices_per_lookup, fixed, round_targets):
    """One batch drawn sample by sample from numpy's GLOBAL RNG in the reference's order
    (generate_dist_input_batch, 'uniform' branch, then generate_random_output_batch).  The CLI's loss
    curves were pinned on these batches; datagen.RandomDataset produces the same ones faster
    (tests/test_datagen.py::test_cli_batches_are_the_dataset_batches) and is what run() uses."""
    ra = np.random
    X = torch.tensor(ra.rand(n, m_den).astype(np.float32))
    lS_o, lS_i = [], []
    for size in ln_emb:
        offs, inds, offset = [], [], 0
        for _ in range(n):
            if fixed:
                k = np.int64(num_indices_per_lookup)
            else:
                r = ra.random(1)
                k = np.int64(np.round(max([1.0], r * min(size, num_indices_per_lookup))))
            r = ra.random(k)
            grp = np.unique(np.round(r * (size - 1)).astype(np.int64))
            offs.append(offset)
            inds += grp.tolist()
            offset += np.int64(grp.size)
        lS_o.append(torch.tensor(offs))
        lS_i.append(torch.tensor(inds))
    if round_targets:
        T = np.round(ra.rand(n, 1).astype(np.float32)).astype(np.float32)
    else:
        T = ra.rand(n, 1).astype(np.float32)
    return X, torch.stack(lS_o), lS_i, torch.tensor(T)


class LRPolicy:
    """Linear warm-up, hold, quadratic decay (LRPolicyScheduler, dlrm_s_pytorch.py:169-203)."""

    def __init__(self, optimizer, warmup, decay_start, decay_steps):
        if decay_start < warmup:
            sys.exit("Learning rate warmup must finish before the decay starts")
        self.opt, self.warmup, self.start, self.steps = optimizer, warmup, decay_start, decay_steps
        self.end = decay_start + decay_steps
        self.base = [g["lr"] for g in optimizer.param_groups]
        self.count, self.last = 0, list(self.base)
        self.step()

    def step(self):
        self.count += 1
        c = self.count
        if c < self.warmup:
            lr = [b * (1.0 - (self.warmup - c) / self.warmup) for b in self.base]
            self.last = lr
        elif self.start <= c < self.end:
            lr = [max(0.0000001, b * ((self.steps - (c - self.start)) / self.steps) ** 2) for b in self.base]
            self.last = lr
        else:
            lr = self.last if self.steps > 0 else self.base
        for g, v in zip(self.opt.param_groups, lr):
            g["lr"] = v


def run(argv=None):
    args = build_parser().parse_args(argv)
    for flag, name in ((args.qr_flag, "--qr-flag"), (args.md_flag, "--md-flag"), (args.save_onnx, "--save-onnx"),
                       (args.mlperf_logging, "--mlperf-logging"), (args.plot_compute_graph, "--plot-compute-graph")):
        if flag:
            sys.exit("ERROR: %s is outside the dlrm_b200 hot path (SURVEY.md section 2)" % name)
    if args.data_generation not in ("random", "synthetic"):
        sys.exit("ERROR: --data-generation=" + args.data_generation + " is not supported (datasets are outside "
                 "the dlrm_b200 hot path; use random or synthetic)")
    if args.quantize_emb_with_bit in [4, 8] or args.quantize_mlp_with_bit != 32:
        sys.exit("ERROR: 4 and 8-bit quantization on GPU is not supported")
    if not torch.cuda.is_available():
        sys.exit("ERROR: dlrm_b200 needs a CUDA device (there is no CPU path); the reference covers CPU runs")
    np.random.seed(args.numpy_rand_seed)
    np.set_printoptions(precision=args.print_precision)
    torch.set_printoptions(precision=args.print_precision)
    torch.manual_seed(args.numpy_rand_seed)
    # one process per GPU under torchrun / mpirun (ext_dist.init_distributed, dlrm_s_pytorch.py:1073-1077)
    rank, world = 0, 1
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        from . import dist as ddist

        backend = args.dist_backend if args.dist_backend else "nccl"
        if backend != "nccl":
            sys.exit("ERROR: --dist-backend=" + backend + " is not supported on GPUs (nccl)")
        if args.local_rank >= 0:
            os.environ.setdefault("LOCAL_RANK", str(args.local_rank))
        rank, world = ddist.init_distributed(backend)
        if rank != 0:      # rank-0-only printing (extend_distributed.py:590-599)
            import builtins

            builtins.print = lambda *a, **k: None
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")) if world > 1 else 0)
    if world > 1:
        torch.cuda.set_device(device)
    print("Using {} GPU(s)...".format(world))

    from . import optim as fused
    from .dlrm_net import DLRM_Net

    ln_bot = np.fromstring(args.arch_mlp_bot, dtype=int, sep="-")
    ln_emb = np.fromstring(args.arch_embedding_size, dtype=int, sep="-")
    m_den = ln_bot[0]
    m_spa = args.arch_sparse_feature_size
    num_fea = ln_emb.size + 1
    m_den_out = ln_bot[ln_bot.size - 1]
    if args.arch_interaction_op == "dot":
        num_int = ((num_fea * (num_fea + 1)) // 2 if args.arch_interaction_itself
                   else (num_fea * (num_fea - 1)) // 2) + m_den_out
    else:
        num_int = num_fea * m_den_out
    ln_top = np.fromstring(str(num_int) + "-" + args.arch_mlp_top, dtype=int, sep="-")
    if m_spa != m_den_out:
        sys.exit("ERROR: arch-sparse-feature-size " + str(m_spa) + " does not match last dim of bottom mlp "
                 + str(m_den_out))
    nbatches = args.num_batches if args.num_batches > 0 else int(np.ceil(args.data_size / args.mini_batch_size))

    # RandomDataset(reset_seed_on_access=True): numpy is re-seeded at the first batch of every epoch, and
    # every batch is drawn in the reference's order (datagen.py; identical batches for identical flags)
    from . import datagen

    train_data, _, test_data, _ = datagen.make_random_data_and_loader(args, ln_emb, m_den)
    nbatches_test = len(test_data)

    def batch(j):
        return datagen.collate_wrapper_random_offset([train_data[j]])

    loss_ws = np.fromstring(args.loss_weights, dtype=float, sep="-") if args.loss_function == "wbce" else None
    dlrm = DLRM_Net(m_spa, ln_emb, ln_bot, ln_top, arch_interaction_op=args.arch_interaction_op,
                    arch_interaction_itself=args.arch_interaction_itself, sigmoid_bot=-1,
                    sigmoid_top=ln_top.size - 2, sync_dense_params=args.sync_dense_params,
                    loss_threshold=args.loss_threshold, ndevices=-1, weighted_pooling=args.weighted_pooling,
                    loss_function=args.loss_function, device=device, gemm=args.gemm,
                    max_batch=args.mini_batch_size, loss_weights=loss_ws)
    optimizer = lr_scheduler = None
    if not args.inference_only:
        if args.optimizer == "sgd":
            optimizer = fused.SGD(dlrm.parameters(), lr=args.learning_rate)
        elif args.optimizer == "rwsadagrad":
            optimizer = fused.RWSAdagrad(dlrm.parameters(), lr=args.learning_rate)
        else:
            sys.exit("ERROR: --optimizer=" + args.optimizer + " is not supported (sgd | rwsadagrad)")
        lr_scheduler = LRPolicy(optimizer, args.lr_num_warmup_steps, args.lr_decay_start_step,
                                args.lr_num_decay_steps)
    if args.debug_mode:                                     # dlrm_s_pytorch.py:1222-1262, :1308-1311
        print("model arch:")
        print("mlp top arch " + str(ln_top.size - 1) + " layers, with input to output dimensions:")
        print(ln_top)
        print("# of interactions")
        print(num_int)
        print("mlp bot arch " + str(ln_bot.size - 1) + " layers, with input to output dimensions:")
        print(ln_bot)
        print("# of features (sparse and dense)")
        print(num_fea)
        print("dense feature size")
        print(m_den)
        print("sparse feature size")
        print(m_spa)
        print("# of embeddings (= # of sparse features) " + str(ln_emb.size) + ", with dimensions "
              + str(m_spa) + "x:")
        print(ln_emb)
        print("initial parameters (weights and bias):")
        for param in dlrm.parameters():
            print(param.detach().cpu().numpy())

    best_acc_test = 0
    skip_upto_epoch = skip_upto_batch = 0
    total_time = total_loss = total_iter = total_samp = 0
    if args.load_model:                                      # dlrm_s_pytorch.py:1399-1456
        print("Loading saved model {}".format(args.load_model))
        ld = torch.load(args.load_model, map_location=device, weights_only=False)
        dlrm.load_state_dict(ld["state_dict"])
        ld_j, ld_k = ld["iter"], ld["epoch"]
        ld_nepochs, ld_nbatches, ld_nbatches_test = ld["nepochs"], ld["nbatches"], ld["nbatches_test"]
        ld_train_loss, ld_total_loss, ld_acc_test = ld["train_loss"], ld["total_loss"], ld["test_acc"]
        if not args.inference_only:
            optimizer.load_state_dict(ld["opt_state_dict"])
            best_acc_test = ld_acc_test
            total_loss = ld_total_loss
            skip_upto_epoch = ld_k
            skip_upto_batch = ld_j
            # dlrm_b200: the schedule resumes at the saved position (the reference's scheduler restarts at step 1)
            for _ in range(ld_k * ld_nbatches + ld_j):
                lr_scheduler.step()
        else:
            args.print_freq = ld_nbatches
            args.test_freq = 0
        print("Saved at: epoch = {:d}/{:d}, batch = {:d}/{:d}, ntbatch = {:d}".format(
            ld_k, ld_nepochs, ld_j, ld_nbatches, ld_nbatches_test))
        print("Training state: loss = {:.6f}".format(ld_train_loss))
        print("Testing state: accuracy = {:3.3f} %".format(ld_acc_test * 100))

    def inference(best_acc):
        """One pass over the test set (inference(), dlrm_s_pytorch.py:759-900): accuracy of round(Z) against the
        targets, every rank's slice gathered first."""
        test_accu = test_samp = 0
        for i in range(nbatches_test):
            if nbatches > 0 and i >= nbatches:
                break
            X_t, lS_o_t, lS_i_t, T_t = datagen.collate_wrapper_random_offset([test_data[i]])
            if world > 1 and X_t.size(0) % world != 0:
                print("Warning: Skiping the batch %d with size %d" % (i, X_t.size(0)))
                continue
            with torch.no_grad():
                Z_t = dlrm(X_t.to(device), lS_o_t, lS_i_t)
            if world > 1:
                import torch.distributed as tdist

                parts = [torch.empty_like(Z_t) for _ in range(world)]
                tdist.all_gather(parts, Z_t.contiguous())
                Z_t = torch.cat(parts)
            S_t, T_n = Z_t.detach().cpu().numpy(), T_t.numpy()
            test_accu += np.sum((np.round(S_t, 0) == T_n).astype(np.uint8))
            test_samp += T_n.shape[0]
        acc = test_accu / test_samp
        metrics = {"nepochs": args.nepochs, "nbatches": nbatches, "nbatches_test": nbatches_test,
                   "state_dict": dlrm.state_dict(), "test_acc": acc}
        is_best = acc > best_acc
        if is_best:
            best_acc = acc
        print(" accuracy {:3.3f} %, best {:3.3f} %".format(acc * 100, best_acc * 100), flush=True)
        return metrics, is_best, best_acc

    def checkpoint(metrics, k, it, train_loss):
        metrics.update(epoch=k, iter=it, train_loss=train_loss, total_loss=total_loss,
                       opt_state_dict=optimizer.state_dict())
        print("Saving model to {}".format(args.save_model))
        if rank == 0:
            torch.save(metrics, args.save_model)

    import contextlib

    prof_ctx = (torch.autograd.profiler.profile(True, use_cuda=True, record_shapes=True)
                if args.enable_profiling else contextlib.nullcontext())
    print("time/loss/accuracy (if enabled):")
    saved = False
    train_loss = 0.0
    with prof_ctx as prof:
        if args.inference_only:
            print("Testing for inference only")
            inference(best_acc_test)
        for k in range(0 if not args.inference_only else args.nepochs, args.nepochs):
            if k < skip_upto_epoch:
                continue
            for j in range(nbatches):
                X, lS_o, lS_i, T = batch(j)       # drawn even when skipped: the generator's order is the reference's
                if j < skip_upto_batch:
                    continue
                if world > 1 and X.size(0) % world != 0:      # dlrm_s_pytorch.py:1565-1570
                    print("Warning: Skiping the batch %d with size %d" % (j, X.size(0)))
                    continue
                torch.cuda.synchronize()
                t1 = time.time()
                Z = dlrm(X.to(device), lS_o, lS_i)
                if world > 1:                               # loss on this rank's batch slice (:1584-1586)
                    nloc = X.size(0) // world
                    T = T[rank * nloc:(rank + 1) * nloc]
                Td = T.to(device)
                if args.loss_function == "wbce":
                    ws = dlrm.loss_ws.to(device)[Td.view(-1).long()].view_as(Td).float()
                    E = (ws * dlrm.loss_fn(Z, Td)).mean()
                else:
                    E = dlrm.loss_fn(Z, Td)
                L = E.detach().cpu().numpy()
                if world > 1 and os.environ.get("DLRM_CLI_GLOBAL_LOSS") == "1":
                    # the reference prints rank 0's slice loss; the mean over the ranks is the single-process loss
                    import torch.distributed as tdist

                    Lg = E.detach().clone()
                    tdist.all_reduce(Lg, op=tdist.ReduceOp.AVG)
                    L = Lg.cpu().numpy()
                optimizer.zero_grad()
                E.backward()
                optimizer.step()
                lr_scheduler.step()
                torch.cuda.synchronize()
                total_time += time.time() - t1
                mbs = T.shape[0]
                total_loss += L * mbs
                total_iter += 1
                total_samp += mbs
                should_print = ((j + 1) % args.print_freq == 0) or (j + 1 == nbatches)
                should_test = (args.test_freq > 0 and args.data_generation in ("dataset", "random")
                               and (((j + 1) % args.test_freq == 0) or (j + 1 == nbatches)))
                if should_print or should_test:
                    gT = 1000.0 * total_time / total_iter if args.print_time else -1
                    train_loss = total_loss / total_samp
                    wall = " ({})".format(time.strftime("%H:%M")) if args.print_wall_time else ""
                    print("Finished {} it {}/{} of epoch {}, {:.2f} ms/it,".format("training", j + 1, nbatches, k, gT)
                          + " loss {:.6f}".format(train_loss) + wall, flush=True)
                    total_time = total_loss = total_iter = total_samp = 0
                if should_test:
                    print("Testing at - {}/{} of epoch {},".format(j + 1, nbatches, k))
                    # (the reference does not carry the best accuracy back to this loop, :1691-1700: every test
                    #  pass that beats the LOADED accuracy saves)
                    metrics, is_best, _ = inference(best_acc_test)
                    if is_best and args.save_model:
                        checkpoint(metrics, k, j + 1, train_loss)
                        saved = True
    if args.save_model and not saved and not args.inference_only:
        # dlrm_b200 addition: the reference only saves after a test pass that improved the accuracy
        # (:1703-1715); without --test-freq it would write nothing, so the final state is saved here
        checkpoint({"nepochs": args.nepochs, "nbatches": nbatches, "nbatches_test": nbatches_test,
                    "state_dict": dlrm.state_dict(), "test_acc": best_acc_test}, args.nepochs, 0, train_loss)
    if args.enable_profiling:                               # dlrm_s_pytorch.py:1795-1805
        import datetime

        stamp = str(datetime.datetime.now()).replace(" ", "_")
        if rank == 0:
            with open("dlrm_s_pytorch" + stamp + "_shape.prof", "w") as f:
                f.write(prof.key_averages(group_by_input_shape=True).table(sort_by="self_cpu_time_total"))
            with open("dlrm_s_pytorch" + stamp + "_total.prof", "w") as f:
                f.write(prof.key_averages().table(sort_by="self_cpu_time_total"))
            prof.export_chrome_trace("dlrm_s_pytorch" + stamp + ".json")
    if not args.inference_only and args.debug_mode:
        print("updated parameters (weights and bias):")
        for param in dlrm.parameters():
            print(param.detach().cpu().numpy())
    return dlrm


if __name__ == "__main__":
    run()
