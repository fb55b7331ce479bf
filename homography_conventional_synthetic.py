#!/usr/bin/env python
"""Drop-in entry point for the reference's `code/homography_conventional_synthetic.py`: the conventional baselines on the
synthetic test set, with the same flags (:50-80), log-dir naming (:85-90), printed lines and results.txt (:185-241).

--method direct runs cv2.findTransformECC (MOTION_HOMOGRAPHY, --num_iterations iterations, eps 1e-10) batched in libudh's
CUDA kernels; --method identity predicts zero displacement and never fails (utils/RANSAC_homography.py:30).  SIFT and ORB
(feature matching + RANSAC) are not built and exit with an error.  The running time is the batch's GPU time (CUDA events
around input preparation, ECC and post-processing) divided by the batch size: a batched figure, not one pair at a time.

New flag: --synthetic N (generate N pairs on the device instead of reading <data_path>/I, I_prime), --seed.
"""
from __future__ import absolute_import, division, print_function

import argparse
import os
import shutil
import sys

import numpy as np

HEIGHT, WIDTH, RHO, PATCH_SIZE = 240, 320, 45, 128          # homography_conventional_synthetic.py:16-19
DATA_PATH = os.environ.get("UDH_DATA_PATH", "/home/tynguyen/pose_estimation/data/synthetic/" + str(RHO) + '/')
LOG_DIR = "../logs/"
AUGMENT_LIST = ['normalize']


def str2bool(s):
    return s.lower() == 'true'


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--mode', type=str, default='test', help='Train or test', choices=['train', 'test'])
    p.add_argument('--method', type=str, default='SIFT', help='RANSAC method', choices=['SIFT', 'ORB', 'identity', 'direct'])
    p.add_argument('--augment_list', nargs='+', default=AUGMENT_LIST, help='List of augmentations')
    p.add_argument('--do_augment', type=float, default=0.5, help='Possibility of augmenting image: color shift, brightness shift...')
    p.add_argument('--num_gpus', type=int, default=2, help='Number of splits')
    p.add_argument('--log_dir', type=str, default=LOG_DIR, help='The log path')
    p.add_argument('--raw_data_path', type=str, default=None)
    p.add_argument('--data_path', type=str, default=DATA_PATH)
    p.add_argument('--I_dir', type=str, default=None)
    p.add_argument('--I_prime_dir', type=str, default=None)
    p.add_argument('--pts1_file', type=str, default=None)
    p.add_argument('--test_pts1_file', type=str, default=None)
    p.add_argument('--gt_file', type=str, default=None)
    p.add_argument('--test_gt_file', type=str, default=None)
    p.add_argument('--filenames_file', type=str, default=None)
    p.add_argument('--test_filenames_file', type=str, default=None)
    p.add_argument('--visual', type=str2bool, default='false', help='Visualize obtained images to debug')
    p.add_argument('--img_w', type=int, default=WIDTH)
    p.add_argument('--img_h', type=int, default=HEIGHT)
    p.add_argument('--patch_size', type=int, default=PATCH_SIZE)
    p.add_argument('--batch_size', type=int, default=128)
    p.add_argument('--max_epoches', type=int, default=1)
    p.add_argument('--num_features', type=int, default=8, help='Number of features used to do RANSAC')
    p.add_argument('--num_iterations', type=int, default=8, help='Number of iterations used to do direct method')
    p.add_argument('--resume', type=str2bool, default='False', help='True: restore the existing model. False: retrain')
    # new
    p.add_argument('--synthetic', type=int, default=0, help='generate this many pairs on the device instead of reading data_path')
    p.add_argument('--seed', type=int, default=0)
    return p


def resolve_paths(args):
    d = args.data_path
    args.I_dir = args.I_dir or d + 'I/'
    args.I_prime_dir = args.I_prime_dir or d + 'I_prime/'
    args.test_pts1_file = args.test_pts1_file or os.path.join(d, 'test_pts1.txt')
    args.test_filenames_file = args.test_filenames_file or os.path.join(d, 'test_synthetic.txt')
    args.test_gt_file = args.test_gt_file or os.path.join(d, 'test_gt.txt')
    prefix = args.method + '/'
    for a in args.augment_list:
        prefix += '_' + a
    prefix += '/' + 'RHO_' + str(RHO) + '_maxfeat_' + str(args.num_features) + '_doaugment_' + str(args.do_augment) + '/'
    args.log_dir = os.path.join(args.log_dir, prefix + args.mode + '/')
    return args


def find_percentile(values):
    """utils/utils.py:655-673: means of the sorted list's thirds."""
    v = sorted(values)
    n = len(v)
    a, b = int(0.3 * n), int(0.6 * n)
    return [float(np.mean(p)) if len(p) else float('nan') for p in (v[:a], v[a:b], v[b:])]


def summarise(h_losses, fails, total_time, num_samples):
    """The five numbers of results.txt (:228-236): samples, mean h_loss, std, failure fraction, seconds per sample."""
    h = np.asarray(h_losses, np.float64)
    return [num_samples, float(np.mean(h)), float(np.std(h)), float(np.sum(np.asarray(fails) != 0)) / num_samples, total_time / num_samples]


def run_batch(method, batch, num_iterations, rho):
    """-> (h_loss [B] float, fail [B] int, GPU seconds) for one Dataloader batch."""
    import torch
    from unsuperviseddeephomographyral2018_b200 import ops
    gt = batch["gt"].contiguous()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if method == 'direct':
        g1, g2 = ops.ecc_prep_u8(batch["I_u8"], batch["I_prime_u8"], batch.get("aug"))
        W, _, _, status = ops.find_homography_ecc(g1, g2, None, num_iterations, 1e-10)
    else:                                                             # identity: W = I, never "not found"
        B = gt.shape[0]
        W = torch.eye(3, device=gt.device).repeat(B, 1, 1).contiguous()
        status = torch.zeros(B, device=gt.device, dtype=torch.int32)
    _, h, fail = ops.ecc_h4p(W, status, batch["pts1"].contiguous(), gt, float(rho))
    e1.record()
    torch.cuda.synchronize()
    return h.cpu().numpy(), fail.cpu().numpy(), e0.elapsed_time(e1) * 1e-3


def test(args):
    import torch
    from unsuperviseddeephomographyral2018_b200 import _lib
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    _lib.require_device()
    if not args.resume:
        shutil.rmtree(args.log_dir, ignore_errors=True)
    os.makedirs(args.log_dir, exist_ok=True)
    num_data = args.synthetic if args.synthetic else dl.count_text_lines(args.test_filenames_file)
    print('===> There are totally %d test files' % num_data)
    batch_size = int(min(num_data, args.batch_size))
    steps = args.max_epoches * int(np.ceil(num_data / batch_size))
    dparams = dl.dataloader_params(data_path=args.data_path, filenames_file=args.test_filenames_file, pts1_file=args.test_pts1_file,
                                   gt_file=args.test_gt_file, mode='test', batch_size=batch_size, img_h=args.img_h, img_w=args.img_w,
                                   patch_size=args.patch_size, augment_list=args.augment_list, do_augment=args.do_augment)
    loader = dl.Dataloader(dparams, shuffle=False, synthetic_pairs=args.synthetic, seed=args.seed, device="cuda")
    h_losses, fails, total_time, num_samples = [], [], 0.0, 0
    for step in range(steps):
        b = loader.next_batch()
        h, f, secs = run_batch(args.method, b, args.num_iterations, RHO)
        total_time += secs
        for i in range(len(h)):
            num_samples += 1
            if f[i] == 1:
                print('===> Fail case 1: Not found homography')
            elif f[i] == 2:
                print('===> Fail case 2:  error > identity')
            h_losses.append(float(h[i])); fails.append(int(f[i]))
        print(' Test| image %d, h_loss %.3f, h_loss_average %.3f, fail %d/%d, time %.4f (batched)'
              % (num_samples - 1, h_losses[-1], np.mean(h_losses), int(np.sum(np.asarray(fails) != 0)), num_samples, secs / len(h)), flush=True)
    line = summarise(h_losses, fails, total_time, num_samples)
    print('==========================================================')
    print('===> H_loss:', line[1], '+/-', line[2])
    print('Running time:', line[4], '(batched: GPU time of a batch / batch size)')
    print('Failure %.3f' % line[3])
    print('output_line:', line)
    with open(os.path.join(args.log_dir, 'results.txt'), 'w') as f:
        np.savetxt(f, [line], delimiter=' ', fmt='%.5f')
        print('===> Wrote results to file %s' % os.path.join(args.log_dir, 'results.txt'))
    print('===> Percentile Values: (30, 60, 100):')
    print(find_percentile(h_losses))
    return line


def main(argv=None):
    args = resolve_paths(build_parser().parse_args(argv))
    print('<==================== Loading raw data ===================>\n')
    print(args.log_dir)
    if args.method in ('SIFT', 'ORB'):
        print('--method %s (feature matching + RANSAC) is not built in this project; use --method direct or identity' % args.method,
              file=sys.stderr)
        return 2
    if args.mode != 'test':
        print('--mode train: the conventional methods have nothing to train', file=sys.stderr)
        return 2
    test(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
