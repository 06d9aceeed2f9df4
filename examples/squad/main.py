"""Fine-tuning BERT on SQuAD with any algorithm — the command line of the reference's examples/squad/main.py:707-990 (the
HuggingFace ``run_squad`` flags plus --algorithm / --async-* / --fuse-optimizer / --set-deterministic / --prof):

    export SQUAD_DIR=/path/to/SQUAD
    python -m bagua_b200.distributed.launch --nproc_per_node=8 examples/squad/main.py --model_type bert \
        --model_name_or_path /models/bert-large-uncased-whole-word-masking --do_train --do_eval --do_lower_case \
        --train_file $SQUAD_DIR/train-v1.1.json --predict_file $SQUAD_DIR/dev-v1.1.json --learning_rate 3e-5 --num_train_epochs 2.0 \
        --max_seq_length 384 --doc_stride 128 --output_dir /tmp/debug_squad/ --per_gpu_eval_batch_size 6 --per_gpu_train_batch_size 6 \
        --algorithm bytegrad

What each part is here (nothing is imported from ``transformers``; there is no network in the build image):

* model — ``bagua_b200.models.BertForQuestionAnswering``.  ``--model_name_or_path`` may be a local HuggingFace-format directory
  (config.json + model.safetensors / pytorch_model.bin, converted on load, tests/test_bert_hf_parity.py); a bare hub name selects the
  architecture (…large… / …base…) with random weights, and says so.
* data — ``squad_utils.py`` next to this file: SQuAD JSON → word-piece features with ``--doc_stride`` windows → n-best decoding →
  exact-match / F1.  ``--tokenizer_name`` (or the model directory) provides ``vocab.txt``; without one a hashing tokenizer is used.
  Without ``--train_file`` / ``--predict_file`` a template-generated SQuAD-format dataset stands in (``--num-synthetic`` paragraphs).
  Features are cached in ``--cache_dir`` (default: next to the data file) like the reference's ``cached_{train,dev}_…`` files.
* optimisation — AdamW (decay on matrices only) with linear warm-up / decay, gradient clipping, gradient accumulation through
  ``model.bagua_ddp.require_backward_grad_sync`` (micro-steps accumulate locally, the last one communicates), or with
  ``--fused-shard --accumulate-in-shard`` in the fp32 gradient shard of the in-bucket optimizer (every micro-step communicates and
  adds its averaged gradient; ``accumulate_grads=True``).  On GPUs parameters are
  bf16 with fp32 master weights inside ``bagua_b200.ops.FusedAdam`` (``--fp16`` is accepted and means this mixed-precision path;
  ``--dtype fp32`` restores full precision; ``--dtype fp16`` trains in real fp16 with dynamic loss scaling, which needs
  ``--fused-shard``: ``ShardedGradScaler`` unscales, detects overflow and skips steps on the device); ``--fused-shard`` moves AdamW
  into the bucket kernels; ``--fuse-optimizer`` uses the
  generic ``bagua.contrib.fuse_optimizer``; ``--load-balance`` batches by non-pad length (LoadBalancingDistributedSampler).
* evaluation — every rank scores a shard of the dev features, rank 0 decodes and writes predictions.json / nbest_predictions.json
  (and null_odds-free v2 handling) to ``--output_dir``; ``--evaluate_during_training`` does so every ``--logging_steps``.
* checkpoints — ``output_dir/checkpoint-<step>/`` every ``--save_steps`` and the final model in ``output_dir``, in HuggingFace
  tensor names, plus optimizer / scheduler state; ``--eval_all_checkpoints`` scores each of them."""
import argparse
import glob
import importlib.util
import json
import logging
import os
import random
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import bagua_b200 as bagua  # noqa: E402
from bagua_b200 import models  # noqa: E402
from bagua_b200.contrib import LoadBalancingDistributedSampler  # noqa: E402
from bagua_b200.parallel.algorithms import Algorithm, q_adam  # noqa: E402
from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, ShardedFusedAdam, ShardedFusedLion,  # noqa: E402
                                                               make_sharded_fused_adam, make_sharded_fused_lion)

_spec = importlib.util.spec_from_file_location("bagua_example_squad_utils", os.path.join(HERE, "squad_utils.py"))
su = importlib.util.module_from_spec(_spec)
sys.modules[_spec.name] = su   # dataclasses defined there need their module registered
_spec.loader.exec_module(su)

log = logging.getLogger("squad")


def parse():
    p = argparse.ArgumentParser(description="bagua_b200 SQuAD fine-tuning")
    a = p.add_argument
    a("--model_type", default="bert", help="only bert is built in")
    a("--model_name_or_path", default="bert-large-uncased-whole-word-masking", help="local HuggingFace-format directory, or a name that selects the architecture")
    a("--output_dir", default="/tmp/debug_squad")
    a("--data_dir", default=None, help="directory with train-v1.1.json / dev-v1.1.json (or the v2.0 files) when the two file flags are not given")
    a("--train_file", default=None)
    a("--predict_file", default=None)
    a("--config_name", default="", help="config.json (file or directory) if not the model's")
    a("--tokenizer_name", default="", help="vocab.txt (file or directory) if not the model's")
    a("--cache_dir", default="", help="where feature caches go (default: next to the data file / output_dir)")
    a("--version_2_with_negative", action="store_true", help="the data has unanswerable questions (SQuAD 2.0)")
    a("--null_score_diff_threshold", type=float, default=0.0)
    a("--max_seq_length", "--max-seq-length", dest="max_seq_length", type=int, default=384)
    a("--doc_stride", type=int, default=128)
    a("--max_query_length", type=int, default=64)
    a("--do_train", action="store_true")
    a("--do_eval", action="store_true")
    a("--evaluate_during_training", action="store_true")
    a("--do_lower_case", action="store_true")
    a("--per_gpu_train_batch_size", "--batch-size", dest="per_gpu_train_batch_size", type=int, default=8)
    a("--per_gpu_eval_batch_size", type=int, default=8)
    a("--learning_rate", "--learning-rate", dest="learning_rate", type=float, default=5e-5)
    a("--gradient_accumulation_steps", type=int, default=1)
    a("--weight_decay", "--weight-decay", dest="weight_decay", type=float, default=0.0)
    a("--adam_epsilon", type=float, default=1e-8)
    a("--max_grad_norm", type=float, default=1.0, help="0 disables clipping")
    a("--num_train_epochs", "--epochs", dest="num_train_epochs", type=float, default=3.0)
    a("--max_steps", type=int, default=-1, help="> 0: total optimizer steps, overrides --num_train_epochs")
    a("--warmup_steps", type=int, default=0)
    a("--n_best_size", type=int, default=20)
    a("--max_answer_length", type=int, default=30)
    a("--verbose_logging", action="store_true")
    a("--lang_id", type=int, default=0, help="accepted for command-line compatibility (XLM only)")
    a("--logging_steps", "--print-freq", dest="logging_steps", type=int, default=500)
    a("--save_steps", type=int, default=500)
    a("--eval_all_checkpoints", action="store_true")
    a("--no_cuda", "--cpu", dest="no_cuda", action="store_true")
    a("--overwrite_output_dir", action="store_true")
    a("--overwrite_cache", action="store_true")
    a("--seed", type=int, default=42)
    a("--fp16", action="store_true", help="accepted: GPUs already train in bf16 with fp32 master weights")
    a("--fp16_opt_level", default="O1", help="accepted for command-line compatibility (apex)")
    a("--server_ip", default="", help="accepted for command-line compatibility (remote debugger)")
    a("--server_port", default="")
    a("--threads", type=int, default=1, help="processes converting examples to features")
    a("--set-deterministic", action="store_true")
    a("--prof", type=int, default=-1, help="profile 10 iterations starting at this one (NVTX + cudaProfilerStart/Stop), then stop")
    a("--algorithm", default="gradient_allreduce", help="gradient_allreduce, bytegrad, decentralized, low_precision_decentralized, qadam, async")
    a("--async-sync-interval", type=int, default=500)
    a("--async-warmup-steps", type=int, default=100)
    a("--fuse-optimizer", action="store_true")
    a("--fused-shard", action="store_true", help="the optimizer inside the bucket kernels (reduce-scatter → update → all-gather)")
    a("--optimizer", default="adamw", choices=["adamw", "lion"],
      help="lion: Lion (betas 0.9, 0.99; give it a 3-10x smaller --learning_rate and a larger --weight_decay than AdamW)")
    a("--accumulate-in-shard", action="store_true",
      help="with --fused-shard and --gradient_accumulation_steps > 1: every micro-step communicates and adds its gradient to the fp32 shard")
    a("--load-balance", action="store_true", help="LoadBalancingDistributedSampler keyed on the number of non-pad tokens")
    a("--dtype", default="bf16", choices=["bf16", "fp32", "fp16"], help="fp16: real fp16 with dynamic loss scaling, needs --fused-shard")
    a("--tiny", action="store_true", help="2-layer model (smoke tests)")
    a("--num-synthetic", type=int, default=256, help="paragraphs of generated SQuAD-format data when no file is given")
    args = p.parse_args()
    if args.model_type != "bert":
        p.error("only --model_type bert is built in")
    if not args.do_train and not args.do_eval:
        args.do_train = args.do_eval = True
    return args


# ---------------------------------------------------------------------------------------------------------------------
# model / tokenizer / data
# ---------------------------------------------------------------------------------------------------------------------
def build_model(args):
    src = args.model_name_or_path
    cfg = None
    if args.config_name:
        cfg = models.BertConfig.from_json_file(args.config_name if os.path.isfile(args.config_name) else os.path.join(args.config_name, "config.json"))
    if os.path.isdir(src) and os.path.isfile(os.path.join(src, "config.json")):
        model, report = models.bert_qa_from_pretrained(src, cfg)
        log.info("loaded %s (missing %s)", src, report["missing"] or "nothing")
        return model
    if cfg is None:
        if args.tiny:
            cfg = models.BertConfig(vocab_size=2048, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, max_position_embeddings=max(args.max_seq_length, 64))
        else:
            cfg = models.bert_large_config() if "large" in src else models.BertConfig()
    log.warning("'%s' is not a local checkpoint directory: %d-layer BERT with RANDOM weights (no network to fetch pretrained ones)", src, cfg.num_hidden_layers)
    return models.BertForQuestionAnswering(cfg)


def data_files(args):
    train, dev = args.train_file, args.predict_file
    if args.data_dir:
        v = "v2.0" if args.version_2_with_negative else "v1.1"
        train = train or os.path.join(args.data_dir, f"train-{v}.json")
        dev = dev or os.path.join(args.data_dir, f"dev-{v}.json")
    return train, dev


def _convert_chunk(job):
    examples, tok, kw, first_id = job
    return su.convert_examples_to_features(examples, tok, first_unique_id=first_id, **kw)


def load_and_cache(args, tokenizer, evaluate: bool, rank: int):
    """Examples + features of the train or dev split; features are built by rank 0 and cached, the other ranks wait and read them."""
    train_file, dev_file = data_files(args)
    path = dev_file if evaluate else train_file
    if path:
        source = path
    else:
        source = su.synthetic_squad(max(args.num_synthetic // 8, 4) if evaluate else args.num_synthetic, seed=2 if evaluate else 1, version_2=args.version_2_with_negative)
    examples = su.read_squad_examples(source, is_training=not evaluate, version_2=args.version_2_with_negative)
    tag = "{}_{}_{}_{}_{}".format("dev" if evaluate else "train", type(tokenizer).__name__, tokenizer.vocab_size, args.max_seq_length, args.doc_stride)
    cache_dir = args.cache_dir or (os.path.dirname(os.path.abspath(path)) if path else args.output_dir)
    cache = os.path.join(cache_dir, f"cached_{tag}_{os.path.basename(path) if path else 'synthetic' + str(args.num_synthetic)}.pt")
    if rank == 0 and (args.overwrite_cache or not os.path.isfile(cache)):
        kw = dict(max_seq_length=args.max_seq_length, doc_stride=args.doc_stride, max_query_length=args.max_query_length, is_training=not evaluate)
        t0 = time.time()
        if args.threads > 1 and len(examples) >= 4 * args.threads:
            import multiprocessing as mp

            step = (len(examples) + args.threads - 1) // args.threads
            jobs = [(examples[i: i + step], tokenizer, kw, 1_000_000_000 + i * 64) for i in range(0, len(examples), step)]
            with mp.get_context("fork").Pool(args.threads) as pool:
                parts = pool.map(_convert_chunk, jobs)
            feats = []
            for part, start in zip(parts, range(0, len(examples), step)):
                for f in part:
                    f.example_index += start
                feats.extend(part)
            for n, f in enumerate(feats):   # one id space again
                f.unique_id = 1_000_000_000 + n
        else:
            feats = su.convert_examples_to_features(examples, tokenizer, **kw)
        os.makedirs(cache_dir, exist_ok=True)
        torch.save(feats, cache + ".tmp")
        os.replace(cache + ".tmp", cache)
        log.info("%d examples → %d features in %.1f s (cached in %s)", len(examples), len(feats), time.time() - t0, cache)
    bagua.barrier()
    feats = torch.load(cache, weights_only=False)
    return examples, feats


# ---------------------------------------------------------------------------------------------------------------------
# evaluation
# ---------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def evaluate(args, model, tokenizer, dev, rank, world, prefix=""):
    examples, feats = load_and_cache(args, tokenizer, evaluate=True, rank=rank)
    t = su.features_to_tensors(feats, is_training=False)
    mine = torch.arange(rank, len(feats), world)
    S = args.max_seq_length
    per_rank = (len(feats) + world - 1) // world
    out = torch.full((per_rank, 1 + 2 * S), -1.0, device=dev)   # [feature index, start logits, end logits]; index −1 = padding row
    model.eval()
    t0 = time.time()
    for lo in range(0, len(mine), args.per_gpu_eval_batch_size):
        idx = mine[lo: lo + args.per_gpu_eval_batch_size]
        start, end = model(t["input_ids"][idx].to(dev), token_type_ids=t["token_type_ids"][idx].to(dev), attention_mask=t["attention_mask"][idx].to(dev))
        out[lo: lo + len(idx), 0] = idx.to(dev).float()
        out[lo: lo + len(idx), 1: 1 + S] = start.float()
        out[lo: lo + len(idx), 1 + S:] = end.float()
    model.train()
    everything = torch.empty(world * per_rank, 1 + 2 * S, device=dev)
    bagua.allgather(out.view(-1), everything.view(-1))
    log.info("  evaluation of %d features took %.1f s", len(feats), time.time() - t0)
    results = None
    if rank == 0:
        rows = everything.cpu()
        logits = {}
        for row in rows[rows[:, 0] >= 0]:
            f = feats[int(row[0])]
            logits[f.unique_id] = (row[1: 1 + S].tolist(), row[1 + S:].tolist())
        preds, nbest = su.compute_predictions(examples, feats, logits, n_best_size=args.n_best_size, max_answer_length=args.max_answer_length,
                                              version_2=args.version_2_with_negative, null_score_diff_threshold=args.null_score_diff_threshold, return_nbest=True)
        os.makedirs(args.output_dir, exist_ok=True)
        with open(os.path.join(args.output_dir, f"predictions_{prefix}.json"), "w") as f:
            json.dump(preds, f, indent=1)
        with open(os.path.join(args.output_dir, f"nbest_predictions_{prefix}.json"), "w") as f:
            json.dump(nbest, f, indent=1)
        results = su.squad_evaluate(examples, preds)
        if args.verbose_logging:
            for ex in examples[:5]:
                log.info("  %s | %s → %r (references %s)", ex.qas_id, ex.question, preds[ex.qas_id], ex.answers[:2])
    return bagua.broadcast_object(results, 0)


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def make_optimizer(args, model, cuda, world):
    decay = [p for _, p in model.named_parameters() if p.ndim > 1]
    no_decay = [p for _, p in model.named_parameters() if p.ndim <= 1]   # biases and LayerNorm
    groups = [{"params": decay, "weight_decay": args.weight_decay}, {"params": no_decay, "weight_decay": 0.0}]
    if args.algorithm == "qadam":
        opt = q_adam.QAdamOptimizer(model.parameters(), lr=args.learning_rate, warmup_steps=100, eps=args.adam_epsilon, weight_decay=args.weight_decay)
        return opt, q_adam.QAdamAlgorithm(opt)
    in_shard = args.accumulate_in_shard and args.gradient_accumulation_steps > 1
    if args.optimizer == "lion":   # the in-bucket Lion also runs without a GPU (all-reduce + FusedLion's CPU update)
        if args.fused_shard and args.algorithm == "gradient_allreduce":
            opt = make_sharded_fused_lion(groups, lr=args.learning_rate, max_grad_norm=args.max_grad_norm if args.max_grad_norm > 0 else None,
                                          loss_scaling=args.dtype == "fp16", accumulate_grads=in_shard)
            return opt, FusedGradientAllReduceAlgorithm(opt)
        opt = bagua.ops.FusedLion(groups, lr=args.learning_rate)
        kw = dict(sync_interval_ms=args.async_sync_interval, warmup_steps=args.async_warmup_steps) if args.algorithm == "async" else {}
        return opt, Algorithm.init(args.algorithm, **kw)
    # without a GPU the in-shard accumulation runs on the fallback (all-reduce + flat AdamW), which accumulates in the model's dtype
    if args.fused_shard and (cuda or in_shard) and args.algorithm == "gradient_allreduce":
        opt = make_sharded_fused_adam(groups, lr=args.learning_rate, eps=args.adam_epsilon, adamw=True,   # buckets are cut per parameter group
                                      max_grad_norm=args.max_grad_norm if args.max_grad_norm > 0 else None,   # clipped inside step()
                                      loss_scaling=args.dtype == "fp16", accumulate_grads=in_shard)
        return opt, FusedGradientAllReduceAlgorithm(opt)
    if cuda and not args.fuse_optimizer:
        opt = bagua.ops.FusedAdam(groups, lr=args.learning_rate, eps=args.adam_epsilon, adamw=True)
    else:
        opt = torch.optim.AdamW(groups, lr=args.learning_rate, eps=args.adam_epsilon)
    kw = dict(sync_interval_ms=args.async_sync_interval, warmup_steps=args.async_warmup_steps) if args.algorithm == "async" else {}
    return opt, Algorithm.init(args.algorithm, **kw)


def save_checkpoint(args, model, optimizer, scheduler, directory, rank):
    state = optimizer.state_dict()   # collective for sharded optimizers: every rank calls it
    if rank == 0:
        models.save_pretrained(model, directory)
        torch.save(state, os.path.join(directory, "optimizer.pt"))
        torch.save(scheduler.state_dict(), os.path.join(directory, "scheduler.pt"))
        with open(os.path.join(directory, "training_args.json"), "w") as f:
            json.dump({k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool, type(None)))}, f, indent=1)
        log.info("saved checkpoint to %s", directory)
    bagua.barrier()   # nobody may look for the files (--eval_all_checkpoints) before rank 0 has finished writing them


def train(args, model, tokenizer, dev, rank, world, cuda):
    examples, feats = load_and_cache(args, tokenizer, evaluate=False, rank=rank)
    t = su.features_to_tensors(feats, is_training=True)
    keys = ["input_ids", "token_type_ids", "attention_mask", "start_positions", "end_positions"]
    dataset = torch.utils.data.TensorDataset(*[t[k] for k in keys])
    if args.load_balance:
        sampler = LoadBalancingDistributedSampler(dataset, complexity_fn=lambda item: int(item[2].sum()), num_replicas=world, rank=rank, shuffle=True)
    else:
        sampler = torch.utils.data.distributed.DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=True, seed=args.seed)
    loader = torch.utils.data.DataLoader(dataset, batch_size=args.per_gpu_train_batch_size, sampler=sampler, drop_last=True, pin_memory=cuda)
    accum = max(args.gradient_accumulation_steps, 1)
    updates_per_epoch = max(len(loader) // accum, 1)
    if args.max_steps > 0:
        total, epochs = args.max_steps, (args.max_steps + updates_per_epoch - 1) // updates_per_epoch
    else:
        total, epochs = int(updates_per_epoch * args.num_train_epochs), int(np.ceil(args.num_train_epochs))
    total = max(total, 1)

    optimizer, algorithm = make_optimizer(args, model, cuda, world)
    model = model.with_bagua([optimizer], algorithm, do_flatten=not args.fuse_optimizer)
    if args.fuse_optimizer:
        optimizer = bagua.contrib.fuse_optimizer(optimizer)
    warm = args.warmup_steps
    scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, lambda s: (s + 1) / max(warm, 1) if s < warm else max(0.0, (total - s) / max(1, total - warm)))

    log.info("***** Running training *****")
    log.info("  Num examples = %d, features = %d", len(examples), len(feats))
    log.info("  Num Epochs = %d", epochs)
    log.info("  Instantaneous batch size per GPU = %d", args.per_gpu_train_batch_size)
    log.info("  Total train batch size (w. parallel, distributed & accumulation) = %d", args.per_gpu_train_batch_size * accum * world)
    log.info("  Gradient Accumulation steps = %d", accum)
    log.info("  Total optimization steps = %d", total)

    def nvtx(name):
        import contextlib

        return torch.cuda.nvtx.range(name) if (cuda and args.prof >= 0) else contextlib.nullcontext()

    sharded = isinstance(optimizer, (ShardedFusedAdam, ShardedFusedLion))
    in_shard = sharded and optimizer.accumulate_grads   # every micro-step communicates; step() consumes the sum in the shard
    grad_norm = None
    # fp16: the scaler hands its device scale to the sharded optimizer, whose step program unscales, votes on overflow and skips
    scaler = bagua.amp.ShardedGradScaler() if args.dtype == "fp16" else None
    skipped = torch.zeros((), device=dev) if scaler is not None else None   # accumulated on the device, read when logging
    step, seen_iters, loss_sum, loss_n, t_log, done = 0, 0, 0.0, 0, time.time(), False
    last_loss = None
    for epoch in range(epochs):
        sampler.set_epoch(epoch)
        if args.algorithm == "async":
            model.bagua_algorithm.resume(model)
        optimizer.zero_grad()
        for it, batch in enumerate(loader):
            if args.prof >= 0 and seen_iters == args.prof and cuda:
                torch.cuda.cudart().cudaProfilerStart()
            ids, tt, am, sp, ep = (x.to(dev, non_blocking=True) for x in batch)
            last_micro = (it + 1) % accum == 0
            model.bagua_ddp.require_backward_grad_sync = last_micro or in_shard     # otherwise earlier micro-steps accumulate locally
            with nvtx(f"iteration {seen_iters}"):
                with nvtx("forward"):
                    loss = model(ids, token_type_ids=tt, attention_mask=am, start_positions=sp, end_positions=ep)[0] / accum
                with nvtx("backward"):
                    (loss if scaler is None else scaler.scale(loss)).backward()
                seen_iters += 1
                if not last_micro:
                    continue
                with nvtx("optimizer.step()"):
                    if args.max_grad_norm > 0 and args.algorithm != "qadam" and not sharded:
                        if args.algorithm in ("gradient_allreduce", "bytegrad"):
                            model.bagua_ddp.wait_pending_comm_ops()   # clip the COMMUNICATED gradient (the reference clips after backward, :262-267)
                        grad_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), args.max_grad_norm)
                    if scaler is not None:
                        scaler.step(optimizer)
                        skipped += optimizer.last_step_skipped
                        scaler.update()
                    else:
                        optimizer.fuse_step() if args.fuse_optimizer else optimizer.step()
                    if sharded:   # the sharded optimizer clipped inside step() (max_grad_norm)
                        grad_norm = optimizer.last_grad_norm
                    scheduler.step()
                    optimizer.zero_grad()
            step += 1
            last_loss = loss.detach() * accum
            if args.logging_steps > 0 and step % args.logging_steps == 0:
                loss_sum, loss_n = loss_sum + last_loss.item(), loss_n + 1
                rate = args.per_gpu_train_batch_size * accum * world * args.logging_steps / max(time.time() - t_log, 1e-9)
                gn = "-" if grad_norm is None else f"{float(grad_norm):.4f}"
                amp = "" if scaler is None else f" loss scale {scaler.get_scale():.0f} skipped {int(skipped.item())}"
                log.info("epoch %d step %d/%d loss %.4f lr %.3g grad norm %s%s %.1f samples/s", epoch, step, total, last_loss.item(), scheduler.get_last_lr()[0], gn, amp,
                         rate)
                if args.evaluate_during_training:
                    res = evaluate(args, model, tokenizer, dev, rank, world, prefix=str(step))
                    log.info("  step %d: exact %.2f f1 %.2f", step, res["exact"], res["f1"])
                t_log = time.time()
            if args.save_steps > 0 and step % args.save_steps == 0:
                save_checkpoint(args, model, optimizer, scheduler, os.path.join(args.output_dir, f"checkpoint-{step}"), rank)
            if args.prof >= 0 and seen_iters >= args.prof + 10:
                if cuda:
                    torch.cuda.cudart().cudaProfilerStop()
                done = True
            if step >= total:
                done = True
            if done:
                break
        if args.algorithm == "async":
            model.bagua_algorithm.abort(model)
        if done:
            break
    model.bagua_ddp.require_backward_grad_sync = True
    return model, optimizer, scheduler, step, (last_loss.item() if last_loss is not None else float("nan"))


def main():
    args = parse()
    cuda = torch.cuda.is_available() and not args.no_cuda
    if cuda:
        torch.cuda.set_device(bagua.get_local_rank())
    bagua.init_process_group()
    rank, world = bagua.get_rank(), bagua.get_world_size()
    logging.basicConfig(format="%(asctime)s - %(levelname)s - %(name)s - %(message)s", datefmt="%m/%d/%Y %H:%M:%S", level=logging.INFO if rank == 0 else logging.WARNING, stream=sys.stdout)
    if os.path.isdir(args.output_dir) and os.listdir(args.output_dir) and args.do_train and not args.overwrite_output_dir and \
            any(n.startswith("checkpoint-") or n in ("model.safetensors", "config.json") for n in os.listdir(args.output_dir)):
        raise SystemExit(f"Output directory ({args.output_dir}) already holds a model. Use --overwrite_output_dir to overcome.")
    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    if args.set_deterministic:
        print("set_deterministic: True")
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
        torch.set_printoptions(precision=10)
    for flag in ("fp16", "server_ip", "lang_id"):
        if getattr(args, flag):
            log.info("--%s is accepted for command-line compatibility and has no effect here", flag)
    dev = torch.device("cuda", bagua.get_local_rank()) if cuda else torch.device("cpu")
    if args.dtype == "fp16" and not (cuda and args.fused_shard and args.algorithm == "gradient_allreduce"):
        raise SystemExit("--dtype fp16 needs a GPU, --fused-shard and --algorithm gradient_allreduce (loss scaling runs in the in-bucket optimizer)")
    if args.optimizer == "lion" and args.algorithm == "qadam":
        raise SystemExit("--optimizer lion does not combine with --algorithm qadam, which brings its own optimizer")
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(args.dtype, torch.float32) if cuda else torch.float32

    model = build_model(args)
    tok_src = args.tokenizer_name or (args.model_name_or_path if os.path.isdir(args.model_name_or_path) else "")
    tokenizer = su.load_tokenizer(tok_src, args.do_lower_case, model.config.vocab_size)
    log.info("tokenizer: %s (%d ids)%s", type(tokenizer).__name__, tokenizer.vocab_size, "" if tok_src else " — no vocab.txt given")
    assert tokenizer.vocab_size <= model.config.vocab_size, "tokenizer has more ids than the model's embedding table"
    assert args.max_seq_length <= model.config.max_position_embeddings, "--max_seq_length exceeds the model's position table"
    model = model.to(dev).to(dtype)
    os.makedirs(args.output_dir, exist_ok=True)

    if args.do_train:
        model, optimizer, scheduler, step, last = train(args, model, tokenizer, dev, rank, world, cuda)
        log.info(" global_step = %s, last loss = %s", step, last)
        save_checkpoint(args, model, optimizer, scheduler, args.output_dir, rank)
    results = {}
    if args.do_eval:
        targets = [("", None)]
        if args.eval_all_checkpoints:
            targets = [(os.path.basename(d).split("-")[-1], d) for d in sorted(glob.glob(os.path.join(args.output_dir, "checkpoint-*")), key=lambda d: int(d.split("-")[-1]))] + targets
        for tag, directory in targets:
            m = model
            if directory is not None:
                m, _ = models.bert_qa_from_pretrained(directory)
                m = m.to(dev).to(dtype)
            res = evaluate(args, m, tokenizer, dev, rank, world, prefix=tag)
            results.update({(f"{k}_{tag}" if tag else k): v for k, v in res.items()})
        log.info("Results: %s", results)
        if rank == 0:
            print(" ".join(f"{k} = {v:.2f}" if isinstance(v, float) else f"{k} = {v}" for k, v in results.items()), flush=True)
    return results


if __name__ == "__main__":
    main()
