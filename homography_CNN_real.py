#!/usr/bin/env python
"""Drop-in entry point for the reference's `code/homography_CNN_real.py` (flags :64-106, train :151-374, TestHomography
:377-640): the real-data (aerial) path of SURVEY §8f-4 —
  * gt-less training: the model is built with gt = None (:268), the loss is photometric (l1_loss by default), no h_loss;
  * --finetune (default True): restore the model trained on synthetic data from --load_model_dir and reset the step to 0
    (:346-353); --resume restores from --save_model_dir instead; checkpoints go to --save_model_dir;
  * test: the ground truth is four hand-picked correspondences per pair; the error is the RMSE of the predicted positions of
    those points on the full-size images, bounded by the identity error (:578-612; real_metrics.correspondence_errors).
Images are 142 x 190 at the network (AREA-resized from 240 x 320 "full" images), patches 128 x 128, RHO = 24 (:17-23).
The arithmetic runs in libudh's sm_90a kernels exactly as for the synthetic path (same engine, one process per GPU).
The classical baselines (RANSAC / direct, --do_report) and --visual (matplotlib windows) are out of scope (DESIGN.md §8).
--mode test --save_visual True (the default) writes the reference's report image of every test sample to results_dir,
named <k>_Unsupervised__loss_<h_loss>.jpg with k global over the ranks, drawn and encoded on the device byte-identical
to cv2 (report.py); the reference's scratch copy /tmp/tmp.jpg is not written.

New flags: --synthetic N (on-device stand-in pairs at the real-data geometry: the aerial set is private), --seed,
--numeric {bf16x3,bf16,fp32}, --max_iterations is the reference's own flag.
"""
from __future__ import absolute_import, division, print_function

import argparse
import os
import shutil
import subprocess
import sys
import time

import numpy as np

import homography_CNN_synthetic as syn

HEIGHT, WIDTH, RHO, PATCH_SIZE = 142, 190, 24, 128          # homography_CNN_real.py:17-20
FULL_HEIGHT, FULL_WIDTH = 240, 320                          # :22-23
DATA_PATH = os.environ.get("UDH_REAL_DATA_PATH", "/home/tynguyen/pose_estimation/data/real/" + str(RHO) + '/')
MAIN_LOG_PATH = '../'
AUGMENT_LIST = ['normalize']


def build_parser():
    s2b = syn.str2bool
    p = argparse.ArgumentParser()
    p.add_argument('--mode', type=str, default='train', choices=['train', 'test'])
    p.add_argument('--loss_type', type=str, default='l1_loss', choices=['h_loss', 'rec_loss', 'ssim_loss', 'l1_loss', 'l1_smooth_loss', 'ncc_loss'])
    p.add_argument('--use_batch_norm', type=s2b, default='False')
    p.add_argument('--leftright_consistent_weight', type=float, default=0)
    p.add_argument('--augment_list', nargs='+', default=AUGMENT_LIST)
    p.add_argument('--do_augment', type=float, default=0.5)
    p.add_argument('--num_gpus', type=int, default=2)
    p.add_argument('--log_dir', type=str, default=MAIN_LOG_PATH + "logs/")
    p.add_argument('--results_dir', type=str, default=MAIN_LOG_PATH + "results/real/report/")
    p.add_argument('--load_model_dir', type=str, default=MAIN_LOG_PATH + "models/synthetic_models/")
    p.add_argument('--save_model_dir', type=str, default=MAIN_LOG_PATH + "models/real_models/")
    p.add_argument('--model_name', type=str, default='model.ckpt')
    p.add_argument('--data_path', type=str, default=DATA_PATH)
    p.add_argument('--I_dir', type=str, default=None)
    p.add_argument('--I_prime_dir', type=str, default=None)
    p.add_argument('--full_I_dir', type=str, default=None)
    p.add_argument('--full_I_prime_dir', type=str, default=None)
    p.add_argument('--pts1_file', type=str, default=None)
    p.add_argument('--test_pts1_file', type=str, default=None)
    p.add_argument('--gt_file', type=str, default=None)                    # GROUND_TRUTH_FILE = None (:37): training has no gt
    p.add_argument('--test_gt_file', type=str, default=None)
    p.add_argument('--filenames_file', type=str, default=None)
    p.add_argument('--test_filenames_file', type=str, default=None)
    p.add_argument('--visual', type=s2b, default='false')
    p.add_argument('--save_visual', type=s2b, default='True',
                   help='--mode test: write every sample\'s report image (JPEG, as the reference\'s) to results_dir')
    p.add_argument('--do_report', type=s2b, default='False')
    p.add_argument('--img_w', type=int, default=WIDTH)
    p.add_argument('--img_h', type=int, default=HEIGHT)
    p.add_argument('--full_img_w', type=int, default=FULL_WIDTH)
    p.add_argument('--full_img_h', type=int, default=FULL_HEIGHT)
    p.add_argument('--patch_size', type=int, default=PATCH_SIZE)
    p.add_argument('--batch_size', type=int, default=128)
    p.add_argument('--max_iterations', type=int, default=150000)
    p.add_argument('--lr', type=float, default=1e-4)
    p.add_argument('--min_lr', type=float, default=.9e-4)
    p.add_argument('--resume', type=s2b, default='False')
    p.add_argument('--retrain', type=s2b, default='False')
    p.add_argument('--finetune', type=s2b, default='True')
    # new
    p.add_argument('--synthetic', type=int, default=0)
    p.add_argument('--seed', type=int, default=0)
    p.add_argument('--numeric', type=str, default='bf16x3', choices=['fp32', 'bf16', 'bf16x3'])
    return p


def resolve_paths(args):
    d = args.data_path
    args.pts1_file = args.pts1_file or os.path.join(d, 'pts1.txt')
    args.filenames_file = args.filenames_file or os.path.join(d, 'train_real.txt')
    args.test_pts1_file = args.test_pts1_file or os.path.join(d, 'test_pts1.txt')
    args.test_filenames_file = args.test_filenames_file or os.path.join(d, 'test_real.txt')
    args.test_gt_file = args.test_gt_file or os.path.join(d, 'test_gt.txt')
    prefix = args.loss_type
    for a in args.augment_list:
        prefix += '_' + a
    args.load_model_dir = os.path.join(args.load_model_dir, prefix)           # :112-115
    args.save_model_dir = os.path.join(args.save_model_dir, prefix)
    args.results_dir = os.path.join(args.results_dir, args.loss_type)
    args.log_dir = os.path.join(args.log_dir, prefix)
    if args.mode == 'test':
        args.log_dir = os.path.join(args.log_dir, prefix + 'test/')
    return args


def loader_params(args, mode, per_gpu):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    test = mode == 'test'
    return dl.extended_dataloader_params(data_path=args.data_path, filenames_file=args.test_filenames_file if test else args.filenames_file,
                                         pts1_file=args.test_pts1_file if test else args.pts1_file,
                                         gt_file=args.test_gt_file if test else args.gt_file, mode=mode, batch_size=per_gpu,
                                         img_h=args.img_h, img_w=args.img_w, patch_size=args.patch_size, augment_list=args.augment_list,
                                         do_augment=args.do_augment, full_img_h=args.full_img_h, full_img_w=args.full_img_w)


def train(args):
    import torch
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en
    rank, world, local, pg = syn.setup(args)
    if rank == 0:
        if not args.resume:
            shutil.rmtree(args.log_dir, ignore_errors=True)
        for d in (args.save_model_dir, args.log_dir, args.results_dir):
            os.makedirs(d, exist_ok=True)
    per_gpu = int(args.batch_size / world)
    loader = dl.Dataloader(loader_params(args, 'train', per_gpu), shuffle=True, synthetic_pairs=args.synthetic, seed=args.seed * 97 + rank, device="cuda", rho=RHO)
    if rank == 0:
        print('===> Train: There are totally %d training files' % loader.num_samples)
        print('===> Decay steps:', en.decay_steps(args.lr, args.min_lr, args.max_iterations))
    eng = en.HomographyEngine(per_gpu, args.patch_size, args.img_h, args.img_w, numeric=args.numeric, seed=args.seed, lr=args.lr,
                              min_lr=args.min_lr, loss_type=args.loss_type, process_group=pg, world_size=world)
    # Restore (:346-353): resume continues a real-data run; finetune starts from the synthetic model with the step reset
    if args.resume and not args.finetune:
        ck, kind = syn.latest_checkpoint(args.save_model_dir, args.model_name)
        if ck:
            syn.restore(eng, ck, kind, reset_step=args.retrain)
    elif args.finetune:
        ck, kind = syn.latest_checkpoint(args.load_model_dir, args.model_name)
        if ck:
            syn.restore(eng, ck, kind, reset_step=True)
            if rank == 0:
                print('===> Finetune from', ck)
        elif rank == 0:
            print('===> --finetune: no checkpoint under %s, training from the seeded initial weights' % args.load_model_dir)
    start = eng.global_step
    sums = dict(rec_loss=0.0, ssim_loss=0.0, l1_loss=0.0, l1_smooth_loss=0.0)
    t0 = time.time()
    step = start
    save_args = argparse.Namespace(model_dir=args.save_model_dir, model_name=args.model_name)
    for step in range(start, start + args.max_iterations):
        out = eng.train_step(loader.next_batch())                             # gt is None: no h_loss, no 4-point metrics
        if step % 100 == 0 or step == start + args.max_iterations - 1:
            d = eng.losses_dict(out)
            if world > 1:
                t = torch.tensor([d[k] for k in sums], device="cuda", dtype=torch.float64)
                torch.distributed.all_reduce(t); t /= world
                d.update(dict(zip(sums, t.tolist())))
            n = 1 if step == start else 100
            for k in sums:
                sums[k] += d[k] * n
            if rank == 0:
                den = step - start + 1
                syn.progress('Train: 1, step %d, rec_loss %4.3f, ssim_loss %.6f. l1_loss %.6f, l1_smooth_loss %.6f, lr %.6f | %.1f pairs/s'
                             % (step, sums["rec_loss"] / den, sums["ssim_loss"] / den, sums["l1_loss"] / den, sums["l1_smooth_loss"] / den,
                                out["lr"], den * args.batch_size / (time.time() - t0)))
        if step and step % 1000 == 0:
            eng.sync_optimizer_state()                                  # collective: Adam's sharded m, v -> complete on every rank
            if rank == 0:
                syn.save(eng, save_args, step)
    eng.sync_optimizer_state()
    if rank == 0:
        syn.save(eng, save_args, step, background=False)
    if world > 1:
        torch.distributed.destroy_process_group()


def test_homography(args):
    import torch
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en, real_metrics as rm, report
    rank, world, local, pg = syn.setup(args)
    if rank == 0:
        for d in (args.log_dir, args.results_dir):
            os.makedirs(d, exist_ok=True)
    num_data = args.synthetic if args.synthetic else dl.count_text_lines(args.test_filenames_file)
    if rank == 0:
        print('===> Test: There are totally %d Test files' % num_data)
    batch = int(min(num_data, args.batch_size))
    per_gpu = max(1, int(batch / world))
    steps = int(np.ceil(num_data / batch))
    loader = dl.Dataloader(loader_params(args, 'test', per_gpu), shuffle=False, synthetic_pairs=args.synthetic, seed=args.seed * 97 + rank + 12345, device="cuda", rho=RHO)
    eng = en.HomographyEngine(per_gpu, args.patch_size, args.img_h, args.img_w, numeric=args.numeric, seed=args.seed, loss_type=args.loss_type,
                              process_group=pg, world_size=world)
    ck, kind = syn.latest_checkpoint(args.save_model_dir, args.model_name)
    if ck:
        syn.restore(eng, ck, kind)
    elif rank == 0:
        print('===> no checkpoint under %s: evaluating the seeded initial weights' % args.save_model_dir)
    h_losses, fails, rec, l1 = [], 0, 0.0, 0.0
    step = 0
    for step in range(steps):
        b = loader.next_batch()
        out = eng.eval_step(b)
        d = eng.losses_dict(out)
        rec += d["rec_loss"]; l1 += d["l1_loss"]
        errs = rm.correspondence_errors(out["pred_h4p"].cpu().numpy(), b["pts1"].cpu().numpy(), b["gt_corr"],
                                        full_img_h=args.full_img_h, img_h=args.img_h, with_points=True)
        for h, ident, failed, _ in errs:
            if failed:
                print("===> Found error > %.3f = RMSE_identity" % ident)
                fails += 1
            h_losses.append(h)
        if args.save_visual:
            # :614-619: every sample, the full-size I on the left, the clicked points and their predicted matches; each
            # rank writes its own samples under their global index
            corr1, corr2 = report.clicked_points(b["gt_corr"])
            n = len(errs)
            names = [report.real_cnn_name(report.global_index(rank, per_gpu, step, args.batch_size, i), errs[i][0]) for i in range(n)]
            report.write(report.render(b, range(n), corr1, corr2, [e[3] for e in errs], prime_left=False), names, args.results_dir)
        if rank == 0:
            syn.progress('Test, h_loss %4.3f, rec_loss %4.3f, l1_loss %4.3f, fail_percent %4.4f'
                         % (float(np.mean(h_losses)), rec / (step + 1), l1 / (step + 1), fails / (step + 1) / per_gpu))
    if world > 1:
        t = torch.tensor([float(np.sum(h_losses)), float(len(h_losses)), float(fails), rec, l1], device="cuda", dtype=torch.float64)
        torch.distributed.all_reduce(t)
        mean_h, fails, rec, l1 = t[0].item() / t[1].item(), t[2].item(), t[3].item() / world, t[4].item() / world
        n = t[1].item()
    else:
        mean_h, n = float(np.mean(h_losses)), len(h_losses)
    if rank == 0:
        print('====> Result for RHO:', RHO, ' loss ', args.loss_type, ' noise ', args.do_augment)
        print('|Steps  |   h_loss   |    l1_loss   |  Fail percent    |')
        print(step, mean_h, l1 / (step + 1), 100.0 * fails / n)
        print('===> Percentile Values: (20, 50, 80, 100):')
        print(syn.find_percentile(h_losses))
        print('======> End! ====================================')
    if world > 1:
        torch.distributed.destroy_process_group()


def main(argv=None):
    args = resolve_paths(build_parser().parse_args(argv))
    print('<==================== Loading data ===================>\n')
    print('===> Load model from (if want) ', args.load_model_dir)
    print('===> Save model to (if want) ', args.save_model_dir)
    rank, world, _ = syn.dist_env()
    if world == 1 and "RANK" not in os.environ:
        import torch
        n = min(args.num_gpus, torch.cuda.device_count()) if torch.cuda.is_available() else 1
        if n > 1:
            from unsuperviseddeephomographyral2018_b200 import build_ext
            build_ext.build()
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
