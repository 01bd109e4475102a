"""`python -m open3dsot_b200.main --cfg cfgs/BAT_Car.yaml [...]`: the reference's command line (main.py:31-93).

Trains with a validation every `--check_val_every_n_epoch` epochs and keeps checkpoints under
`<log_dir>/lightning_logs/version_N/checkpoints/`; `--checkpoint x.ckpt` resumes from a checkpoint of ours or of the
reference's; `--checkpoint x.ckpt --test` evaluates it on `test_split` and prints (and writes to `<log_dir>/test.json`) its
Success and Precision.  Every flag, defaults included, overrides the config's key of the same name, as in the reference.
Under `torchrun` every process trains on its own GPU and the evaluations are split across them."""
import argparse
import json
import os
import sys


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m open3dsot_b200.main")
    p.add_argument('--batch_size', type=int, default=100, help='input batch size')
    p.add_argument('--epoch', type=int, default=60, help='number of epochs')
    p.add_argument('--save_top_k', type=int, default=-1, help='save top k checkpoints')
    p.add_argument('--check_val_every_n_epoch', type=int, default=1, help='check_val_every_n_epoch')
    p.add_argument('--workers', type=int, default=10, help='accepted for compatibility; batches are built on the GPU')
    p.add_argument('--cfg', type=str, help='the config_file')
    p.add_argument('--checkpoint', type=str, default=None, help='checkpoint location')
    p.add_argument('--log_dir', type=str, default=None, help='log location')
    p.add_argument('--test', action='store_true', default=False, help='test mode')
    p.add_argument('--preloading', action='store_true', default=False, help='preload dataset into memory')
    p.add_argument('--precision', choices=('fp32', 'bf16'), default='fp32',
                   help='--test: operand precision of the tensor-core layers (bf16: BF16 operands, FP32 accumulation); '
                        'training is fp32 only')
    p.add_argument('--train_precision', choices=('fp32', 'bf16'), default='fp32',
                   help='training: operand precision of the tensor-core GEMMs of the training steps (bf16: BF16 operands, FP32 '
                        'accumulation, fp32 weights and optimizer state); validation runs in fp32; --test ignores it')
    return p.parse_args(argv)


def parse_config(argv=None):
    """The config file with every flag written over it (main.py:45-49)."""
    from .config import load_config
    args = parse_args(argv)
    if args.cfg is None:
        raise SystemExit("--cfg is required")
    return load_config(args.cfg, vars(args))


def main(argv=None):
    import torch

    from . import ddp
    from .checkpoint import load_lightning_checkpoint
    from .datasets import get_dataset
    from .models import get_model
    from .trainer import Trainer, check_supported, load_weights

    cfg = parse_config(argv)
    if not cfg.test:
        check_supported(cfg)
    rank, world, local = ddp.init_distributed()
    if world > 1:
        ddp.pin_to_gpu_numa_node(local)
    torch.cuda.set_device(local)
    try:
        log_dir = cfg.log_dir or os.getcwd()
        torch.manual_seed(0)
        model = get_model(cfg.net_model)(cfg).cuda()
        if cfg.test:
            if cfg.checkpoint is not None:
                load_weights(model, load_lightning_checkpoint(cfg.checkpoint)["state_dict"])
            tracklets = get_dataset(cfg, type='test', split=cfg.test_split)
            from .tracking.evaluate import evaluate_sharded
            res = evaluate_sharded(model, tracklets, slots=32, seed=0, precision=cfg.precision)
            out = {"checkpoint": cfg.checkpoint, "split": cfg.test_split, "success": res["success"],
                   "precision": res["precision"], "frames": res["frames"]}
            if rank == 0:
                print(json.dumps(out), flush=True)
                os.makedirs(log_dir, exist_ok=True)
                with open(os.path.join(log_dir, "test.json"), "w") as f:
                    json.dump(out, f)
            return out
        train = get_dataset(cfg, type=cfg.train_type, split=cfg.train_split, device=torch.device("cuda", local))
        val = get_dataset(cfg, type='test', split=cfg.val_split)
        trainer = Trainer(model, cfg, train.data, val, log_dir)        # the trainer's sampler reuses the device tracklets
        if cfg.checkpoint is not None:
            trainer.resume(cfg.checkpoint)
        return trainer.fit()
    finally:
        if torch.distributed.is_initialized():
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1:])
