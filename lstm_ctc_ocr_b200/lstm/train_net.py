"""CLI with the reference's flags (lstm/train_net.py:17-48): ``python -m lstm_ctc_ocr_b200.lstm.train_net --network=LSTM_train
--cfg=./lstm/lstm.yml --restore=0`` (what train.sh runs).  Under torchrun it trains data-parallel (NCCL)."""
import argparse
import os
import pprint
import sys

import numpy as np


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Train a lstm network")
    p.add_argument("--gpu", dest="gpu_id", help="GPU device id to use [0]", default=0, type=int)
    p.add_argument("--iters", dest="max_iters", help="number of iterations to train", default=1000000, type=int)
    p.add_argument("--cfg", dest="cfg_file", help="optional config file", default=None, type=str)
    p.add_argument("--pre_train", dest="pre_train", help="pre trained model", default=None, type=str)
    p.add_argument("--rand", dest="randomize", help="randomize (do not use a fixed seed)", action="store_true")
    p.add_argument("--network", dest="network_name", help="name of the network", default=None, type=str)
    p.add_argument("--set", dest="set_cfgs", help="set config keys", default=None, nargs=argparse.REMAINDER)
    p.add_argument("--restore", dest="restore", help="restore or not", default=0, type=int)
    if argv is None and len(sys.argv) == 1:
        p.print_help()
    return p.parse_args(argv)


def main(argv=None):
    import torch
    from ..lib.lstm.config import AttrDict, cfg, cfg_from_file, cfg_from_list, get_log_dir, get_output_dir
    from ..lib.lstm.train import train_net
    from ..lib.networks.factory import get_network
    args = parse_args(argv)
    print("Called with args:")
    print(args)
    if args.cfg_file is not None:
        cfg_from_file(args.cfg_file)
    if args.set_cfgs is not None:
        cfg_from_list(args.set_cfgs)
    if not torch.cuda.is_available():
        from .._lib import CrnnError
        raise CrnnError("train_net needs a CUDA device (sm_90a); there is no CPU fallback")
    if "LOCAL_RANK" in os.environ:                       # torchrun: one process per GPU, NCCL gradient all-reduce
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    else:
        torch.cuda.set_device(args.gpu_id if torch.cuda.device_count() > args.gpu_id else 0)
    print("Using config:")
    pprint.pprint(cfg)
    if not args.randomize:
        np.random.seed(cfg.RNG_SEED)
    output_network_name = args.network_name.split("_")[-1]
    imgdb = AttrDict(path="./data/train_4_6.tfrecords", name="lstm_" + output_network_name, val_path="./data/val.tfrecords")
    output_dir = get_output_dir(imgdb, None)
    log_dir = get_log_dir(imgdb)
    print("Output will be saved to `{:s}`".format(output_dir))
    print("Logs will be saved to `{:s}`".format(log_dir))
    network = get_network(args.network_name)
    print("Use network `{:s}` in training".format(args.network_name))
    train_net(network, imgdb, pre_train=args.pre_train, output_dir=output_dir, log_dir=log_dir, max_iters=args.max_iters,
              restore=bool(int(args.restore)))


if __name__ == "__main__":
    main()
