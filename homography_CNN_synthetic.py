#!/usr/bin/env python
"""Drop-in entry point for the reference's `code/homography_CNN_synthetic.py` (flags :49-85, train() :151-389,
TestHomography :391-580): same flags, modes, printed metrics and checkpoint cadence; the arithmetic runs in libudh's
sm_90a CUDA kernels, one process per GPU (torchrun) with one NCCL gradient allreduce per step.

New flags: --synthetic N (generate N pairs on the device instead of reading <data_path>/I, I_prime — MS-COCO is not
available offline), --seed, --numeric {bf16x3,bf16,fp32} (default bf16x3: the parity-certified tensor-core mode),
--num_total_steps (the reference hard-codes 150000, :161).
"""
from __future__ import absolute_import, division, print_function

import argparse
import glob
import os
import shutil
import subprocess
import sys
import time

import numpy as np

HEIGHT, WIDTH, RHO, PATCH_SIZE = 240, 320, 45, 128          # homography_CNN_synthetic.py:14-17
DATA_PATH = os.environ.get("UDH_DATA_PATH", "/home/tynguyen/pose_estimation/data/synthetic/" + str(RHO) + '/')
MAIN_LOG_PATH = '../'
LOG_DIR = MAIN_LOG_PATH + "logs/"
MODEL_DIR = MAIN_LOG_PATH + "models/synthetic_models"
RESULTS_DIR = MAIN_LOG_PATH + "results/synthetic/report/"
AUGMENT_LIST = ['normalize']


def str2bool(s):
    return s.lower() == 'true'


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--mode', type=str, default='train', help='Train or test', choices=['train', 'test'])
    p.add_argument('--loss_type', type=str, default='l1_loss', help='Loss type',
                   choices=['h_loss', 'rec_loss', 'ssim_loss', 'l1_loss', 'l1_smooth_loss', 'ncc_loss'])
    p.add_argument('--use_batch_norm', type=str2bool, default='False', help='Use batch_norm?')
    p.add_argument('--leftright_consistent_weight', type=float, default=0)
    p.add_argument('--augment_list', nargs='+', default=AUGMENT_LIST, help='List of augmentations')
    p.add_argument('--do_augment', type=float, default=0.5)
    p.add_argument('--num_gpus', type=int, default=2, help='Number of splits')
    p.add_argument('--log_dir', type=str, default=LOG_DIR)
    p.add_argument('--results_dir', type=str, default=RESULTS_DIR)
    p.add_argument('--model_dir', type=str, default=MODEL_DIR)
    p.add_argument('--model_name', type=str, default='model.ckpt')
    p.add_argument('--data_path', type=str, default=DATA_PATH)
    p.add_argument('--I_dir', type=str, default=None)
    p.add_argument('--I_prime_dir', type=str, default=None)
    p.add_argument('--pts1_file', type=str, default=None)
    p.add_argument('--test_pts1_file', type=str, default=None)
    p.add_argument('--gt_file', type=str, default=None)
    p.add_argument('--test_gt_file', type=str, default=None)
    p.add_argument('--filenames_file', type=str, default=None)
    p.add_argument('--test_filenames_file', type=str, default=None)
    p.add_argument('--visual', type=str2bool, default='false')
    p.add_argument('--save_visual', type=str2bool, default='True')
    p.add_argument('--img_w', type=int, default=WIDTH)
    p.add_argument('--img_h', type=int, default=HEIGHT)
    p.add_argument('--patch_size', type=int, default=PATCH_SIZE)
    p.add_argument('--batch_size', type=int, default=128)
    p.add_argument('--max_epoches', type=int, default=150)
    p.add_argument('--lr', type=float, default=1e-4, help='Max learning rate')
    p.add_argument('--min_lr', type=float, default=.9e-4, help='Min learning rate')
    p.add_argument('--resume', type=str2bool, default='False')
    p.add_argument('--retrain', type=str2bool, default='False')
    # new
    p.add_argument('--synthetic', type=int, default=0, help='generate this many pairs on the device instead of reading data_path')
    p.add_argument('--seed', type=int, default=0)
    # bf16x3 = wgmma tensor cores with two-limb (fp32-grade) operands: the parity-certified default.  bf16 = single-pass
    # throughput mode (tenths of a pixel from fp32 on a trained net), fp32 = CUDA cores.
    p.add_argument('--numeric', type=str, default='bf16x3', choices=['fp32', 'bf16', 'bf16x3'])
    p.add_argument('--num_total_steps', type=int, default=150000)
    return p


def resolve_paths(args):
    """Defaults derived from data_path (homography_CNN_synthetic.py:20-33) and the directory munging of :88-114."""
    d = args.data_path
    args.I_dir = args.I_dir or d + 'I/'
    args.I_prime_dir = args.I_prime_dir or d + 'I_prime/'
    args.pts1_file = args.pts1_file or os.path.join(d, 'pts1.txt')
    args.filenames_file = args.filenames_file or os.path.join(d, 'train_synthetic.txt')
    args.gt_file = args.gt_file or os.path.join(d, 'gt.txt')
    args.test_pts1_file = args.test_pts1_file or os.path.join(d, 'test_pts1.txt')
    args.test_filenames_file = args.test_filenames_file or os.path.join(d, 'test_synthetic.txt')
    args.test_gt_file = args.test_gt_file or os.path.join(d, 'test_gt.txt')
    prefix = args.loss_type
    for a in args.augment_list:
        prefix += '_' + a
    if args.mode == 'test':
        args.log_dir = os.path.join(args.log_dir, prefix + 'test/')
    args.model_dir = os.path.join(args.model_dir, prefix)
    args.log_dir = os.path.join(args.log_dir, prefix)
    if args.mode == 'test':
        args.log_dir = os.path.join(args.log_dir, prefix + 'test/')        # applied twice in the reference (:94-100)
    return args


def make_dirs(args, rank):
    if rank != 0:
        return
    if not args.resume:
        shutil.rmtree(args.log_dir, ignore_errors=True)
    for d in (args.model_dir, args.log_dir, args.results_dir):
        os.makedirs(d, exist_ok=True)


def latest_checkpoint(model_dir, model_name):
    """The reference saves TF checkpoints to model_dir + model_name (string concat, :360) and restores from
    tf.train.latest_checkpoint(model_dir) (:315).  Here both sides use  <model_dir>/<model_name>-<step>  as the prefix of a
    TensorFlow V2 bundle (.index + .data-00000-of-00001, written without TensorFlow: tf_checkpoint.py) plus the `checkpoint`
    state file; `.pt` files of round 1 are still found.  Returns (path, kind)."""
    from unsuperviseddeephomographyral2018_b200 import tf_checkpoint as tfc
    p = tfc.latest_checkpoint(model_dir)
    if p and os.path.exists(p + ".index"):
        return p, "tf"
    c = glob.glob(os.path.join(model_dir, model_name + "-*.index"))
    if c:
        return max(c, key=lambda f: int(f.rsplit("-", 1)[1][:-6]))[:-6], "tf"
    c = glob.glob(os.path.join(model_dir, model_name + "-*.pt"))
    return (max(c, key=lambda f: int(f.rsplit("-", 1)[1][:-3])), "pt") if c else (None, None)


def restore(eng, ck, kind, reset_step=False):
    import torch
    if kind == "tf":
        eng.load_tf_checkpoint(ck, reset_step=reset_step)
    else:
        eng.load_state_dict(torch.load(ck, map_location="cpu"), reset_step=reset_step)


_save_thread = None


def wait_for_save():
    """Join the checkpoint writer of the previous save() (call before exiting or before reading model_dir)."""
    global _save_thread
    if _save_thread is not None:
        _save_thread.join()
        _save_thread = None


def save(eng, args, step, background=True):
    """train_saver.save(sess, model_dir + model_name, global_step) (:360).  The state is copied to the host here; the 410 MB
    bundle (parameters + Adam slots) is encoded and written by a thread while training continues."""
    global _save_thread
    import threading
    from unsuperviseddeephomographyral2018_b200 import tf_checkpoint as tfc
    prefix = os.path.join(args.model_dir, "%s-%d" % (args.model_name, step))
    wait_for_save()
    variables = eng.snapshot_tf_variables()

    def write():
        tfc.write_checkpoint(prefix, variables)
        tfc.update_checkpoint_state(args.model_dir, prefix, keep=5)             # Saver(max_to_keep=5), :303

    if background:
        _save_thread = threading.Thread(target=write, name="udh-checkpoint-writer")
        _save_thread.start()
    else:
        write()


def dist_env():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def setup(args):
    import torch
    import torch.distributed as dist
    rank, world, local = dist_env()
    torch.cuda.set_device(local)
    pg = None
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_MAX_CTAS", "32")                  # bound the allreduce kernel to the SMs the conv4_x backward leaves free
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        pg = dist.group.WORLD
    return rank, world, local, pg


def progress(msg):
    print(msg, flush=True)


def train(args):
    import torch
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en
    rank, world, local, pg = setup(args)
    make_dirs(args, rank)
    per_gpu = int(args.batch_size / world)                               # :219 batch_size / num_gpus per tower
    dparams = dl.dataloader_params(data_path=args.data_path, filenames_file=args.filenames_file, pts1_file=args.pts1_file,
                                   gt_file=args.gt_file, mode='train', batch_size=per_gpu, img_h=args.img_h, img_w=args.img_w,
                                   patch_size=args.patch_size, augment_list=args.augment_list, do_augment=args.do_augment)
    loader = dl.Dataloader(dparams, shuffle=True, synthetic_pairs=args.synthetic, seed=args.seed * 97 + rank, device="cuda")
    if rank == 0:
        print('===> Train: There are totally %d training files' % loader.num_samples)
        print('args lr:', args.lr, args.min_lr)
        print('===> Decay steps:', en.decay_steps(args.lr, args.min_lr))
    eng = en.HomographyEngine(per_gpu, args.patch_size, args.img_h, args.img_w, numeric=args.numeric, seed=args.seed,
                              lr=args.lr, min_lr=args.min_lr, loss_type=args.loss_type, process_group=pg, world_size=world)
    if args.resume:
        ck, kind = latest_checkpoint(args.model_dir, args.model_name)
        if ck:
            restore(eng, ck, kind, reset_step=args.retrain)                                        # :314-317
    start = eng.global_step
    if rank == 0:
        print('===> Start step:', start)
    sums = dict(h_loss=0.0, rec_loss=0.0, ssim_loss=0.0, l1_loss=0.0, l1_smooth_loss=0.0, ncc_loss=0.0)
    writer = None
    if rank == 0:
        from unsuperviseddeephomographyral2018_b200 import tb_events
        writer = tb_events.SummaryWriter(args.log_dir)                  # tf.summary.FileWriter(args.log_dir, ...), :300
    t0 = time.time()
    step = start
    for step in range(start, start + args.num_total_steps):
        out = eng.train_step(loader.next_batch())
        if step % 100 == 0 or step == start + args.num_total_steps - 1:
            d = eng.losses_dict(out)                                     # D2H only when something is printed
            if world > 1:                                                # mean of tower losses (:279-284)
                t = torch.tensor([d[k] for k in sums], device="cuda", dtype=torch.float64)
                torch.distributed.all_reduce(t); t /= world
                d.update(dict(zip(sums, t.tolist())))
            n = 1 if step == start else 100
            for k in sums:
                sums[k] += d[k] * n
            if rank == 0:
                den = step - start + 1
                if args.loss_type == "l1_loss":
                    progress('Train: 1, step %d, h_loss %4.3f, l1_loss %.6f, l1_smooth_loss %.6f, lr %.6f | %.1f pairs/s'
                             % (step, sums["h_loss"] / den, sums["l1_loss"] / den, sums["l1_smooth_loss"] / den, out["lr"],
                                den * args.batch_size / (time.time() - t0)))
                else:
                    progress('Train: 1, step %d, h_loss %4.3f, rec_loss %4.3f, ssim_loss %.6f. l1_loss %.6f, l1_smooth_loss %.6f, ncc_loss %.6f, lr %.6f | %.1f pairs/s'
                             % (step, sums["h_loss"] / den, sums["rec_loss"] / den, sums["ssim_loss"] / den, sums["l1_loss"] / den,
                                sums["l1_smooth_loss"] / den, sums["ncc_loss"] / den, out["lr"], den * args.batch_size / (time.time() - t0)))
        if step % 1000 == 0:                                            # TensorBoard scalars, :285-293,356-358
            d = eng.losses_dict(out)
            if world > 1:
                t = torch.tensor([d[k] for k in sums], device="cuda", dtype=torch.float64)
                torch.distributed.all_reduce(t); t /= world
                d.update(dict(zip(sums, t.tolist())))
            if writer:
                sc = {"Losses/Learning_rate": out["lr"]}
                sc.update({"Losses/Total_" + k: d[k] for k in sums})
                writer.add_scalars(sc, step)
        if step and step % 1000 == 0:                                   # :359-360
            eng.sync_optimizer_state()                                  # collective: Adam's sharded m, v -> complete on every rank
            if rank == 0:
                save(eng, args, step)
    eng.sync_optimizer_state()
    if rank == 0:
        save(eng, args, step, background=False)                         # :389
    if world > 1:
        torch.distributed.destroy_process_group()


def find_percentile(values):
    """utils/utils.py:655-673: means of the sorted list's thirds (printed as '(20, 50, 80, 100)' by the reference)."""
    v = sorted(values)
    n = len(v)
    a, b = int(0.3 * n), int(0.6 * n)
    parts = [v[:a], v[a:b], v[b:]]
    return [float(np.mean(p)) if len(p) else float('nan') for p in parts]


def test_homography(args):
    import torch
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en
    rank, world, local, pg = setup(args)
    make_dirs(args, rank)
    num_data = args.synthetic if args.synthetic else dl.count_text_lines(args.test_filenames_file)
    if rank == 0:
        print('===> Test: There are totally %d Test files' % num_data)
    batch = int(min(num_data, args.batch_size))
    per_gpu = max(1, int(batch / world))
    steps = 3 * int(np.ceil(num_data / args.batch_size))                # "Test 3 epoches" (:400-401)
    dparams = dl.dataloader_params(data_path=args.data_path, filenames_file=args.test_filenames_file, pts1_file=args.test_pts1_file,
                                   gt_file=args.test_gt_file, mode='test', batch_size=per_gpu, img_h=args.img_h, img_w=args.img_w,
                                   patch_size=args.patch_size, augment_list=args.augment_list, do_augment=args.do_augment)
    loader = dl.Dataloader(dparams, shuffle=True, synthetic_pairs=args.synthetic, seed=args.seed * 97 + rank + 12345, device="cuda")
    eng = en.HomographyEngine(per_gpu, args.patch_size, args.img_h, args.img_w, numeric=args.numeric, seed=args.seed,
                              loss_type=args.loss_type, process_group=pg, world_size=world)
    ck, kind = latest_checkpoint(args.model_dir, args.model_name)
    if rank == 0:
        print(args.model_dir)
    if ck:
        restore(eng, ck, kind)
    elif rank == 0:
        print('===> no checkpoint under %s: evaluating the seeded initial weights' % args.model_dir)
    tot = dict(h=0.0, rec=0.0, ssim=0.0, l1=0.0, fail=0.0)
    h_losses_array = []
    step = 0
    for step in range(steps):
        out = eng.eval_step(loader.next_batch())
        d = eng.losses_dict(out)
        vals = torch.tensor([d["bounded_h_loss"], d["rec_loss"], d["ssim_loss"], d["l1_loss"], d["num_fail"]], device="cuda", dtype=torch.float64)
        if world > 1:
            torch.distributed.all_reduce(vals); vals[:4] /= world
        h, rec, ssim, l1, fail = vals.tolist()
        tot["h"] += h; tot["rec"] += rec; tot["ssim"] += ssim; tot["l1"] += l1; tot["fail"] += fail
        h_losses_array.append(h)
        if step % 10 == 0 and rank == 0:
            print('===> This iteration num Fail: %d \n' % fail)
            progress('Test, h_loss %4.3f, rec_loss %4.3f, ssim_loss %4.3f, l1_loss %4.3f, fail_percent %4.4f'
                     % (tot["h"] / (step + 1), tot["rec"] / (step + 1), tot["ssim"] / (step + 1), tot["l1"] / (step + 1),
                        tot["fail"] / (step + 1) / args.batch_size))
    if rank == 0:
        print('====> Result for RHO:', RHO, ' loss ', args.loss_type, ' noise ', args.do_augment)
        print('|Steps  |   h_loss   |    l1_loss   |  Fail percent    |')
        print(step, tot["h"] / (step + 1), tot["l1"] / (step + 1), 100 * tot["fail"] / (step + 1) / args.batch_size)
        print('===> Percentile Values: (20, 50, 80, 100):')
        print(find_percentile(h_losses_array))
        print('======> End! ====================================')
    if world > 1:
        torch.distributed.destroy_process_group()


def main(argv=None):
    args = resolve_paths(build_parser().parse_args(argv))
    print('<==================== Loading data ===================>\n')
    rank, world, _ = dist_env()
    if world == 1 and "RANK" not in os.environ:
        import torch
        n = min(args.num_gpus, torch.cuda.device_count()) if torch.cuda.is_available() else 1
        if n > 1:
            # build libudh.so once here, before N ranks import the package at the same moment (build_ext also holds a file lock)
            from unsuperviseddeephomographyral2018_b200 import build_ext
            build_ext.build()
            # the reference builds num_gpus in-graph towers; here: one process per GPU
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
                   "--master-port", str(29500 + os.getpid() % 1000), os.path.abspath(__file__)] + (argv if argv is not None else sys.argv[1:])
            return subprocess.call(cmd)
    if args.mode == 'train':
        train(args)
    else:
        test_homography(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
