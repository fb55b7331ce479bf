#!/usr/bin/env python
"""Drop-in entry point for the reference's `code/homography_conventional_real.py`: the conventional baselines on the real
(aerial) test set, scored on four hand-clicked correspondences per pair, with the same flags (:60-95), log-dir and
results-dir naming (:100-107), printed lines, results.txt and h_losses.pkl (:213-281).

--method direct runs cv2.findTransformECC (MOTION_HOMOGRAPHY, --num_iterations iterations, eps 1e-10) batched in libudh's
CUDA kernels on the full-size (240 x 320) gray planes the reference hands over, cvtColor(denorm_img(full I_aug)); the
loader reads and prepares the batch on the device.  --method identity predicts W = I and never fails.  The metric
(udh_ecc_corr_h4p) follows the reference: the clicked points are halved onto the full-size images, mapped through W (not
inverted), clamped to +-80 px and scored by their RMSE; a sample fails when ECC raised (1) or when the identity does
better (2, scored with the identity error).  SIFT and ORB (feature matching + RANSAC) are not built and exit with an
error, as does --mode train.  --save_visual True (the default) writes the reference's report image of every pair to
results_dir as <k>_loss_<h_loss>.jpg: the full-size images, the clicked points and pred_h4p + corr1 with the clamped
pred_h4p, drawn and encoded on the device byte-identical to cv2 (report.py); the reference's scratch copy tmp.jpg is not
written.  --visual and --artifact_mode noise are accepted and do nothing.  The running time is the batch's GPU time (CUDA events around input preparation, ECC and the metric)
divided by the batch size: a batched figure, not one pair at a time.

New flags: --synthetic N (N full-size pairs generated on the device instead of reading <data_path>, with four
correspondences per pair from the generating homography, in the reference's 2x clicked frame), --seed.
"""
from __future__ import absolute_import, division, print_function

import argparse
import os
import pickle
import shutil
import sys

import numpy as np

HEIGHT, WIDTH, RHO, PATCH_SIZE = 142, 190, 24, 128           # homography_conventional_real.py:17-20
FULL_HEIGHT, FULL_WIDTH = 240, 320                           # :22-23
DATA_PATH = os.environ.get("UDH_REAL_DATA_PATH", "/home/tynguyen/pose_estimation/data/real/" + str(RHO) + '/')
LOG_DIR = "../logs/real_logs"
RESULTS_DIR = "../results/real/"
AUGMENT_LIST = ['normalize']


def str2bool(s):
    return s.lower() == 'true'


def build_parser():
    d = DATA_PATH
    p = argparse.ArgumentParser()
    p.add_argument('--mode', type=str, default='test', help='Train or test', choices=['train', 'test'])
    p.add_argument('--method', type=str, default='SIFT', help='methods', choices=['SIFT', 'ORB', 'identity', 'direct'])
    p.add_argument('--augment_list', nargs='+', default=AUGMENT_LIST, help='List of augmentations')
    p.add_argument('--do_augment', type=float, default=0.5, help='Possibility of augmenting image: color shift, brightness shift...')
    p.add_argument('--num_gpus', type=int, default=2, help='Number of splits')
    p.add_argument('--log_dir', type=str, default=LOG_DIR, help='The log path')
    p.add_argument('--results_dir', type=str, default=RESULTS_DIR, help='The dir to store images for report')
    p.add_argument('--data_path', type=str, default=d, help='The raw data path.')
    p.add_argument('--I_dir', type=str, default=d + 'I/')
    p.add_argument('--I_prime_dir', type=str, default=d + 'I_prime/')
    p.add_argument('--full_I_dir', type=str, default=d + 'FULL_I/')
    p.add_argument('--full_I_prime_dir', type=str, default=d + 'FULL_I_prime/')
    p.add_argument('--pts1_file', type=str, default=os.path.join(d, 'pts1.txt'))
    p.add_argument('--test_pts1_file', type=str, default=None)
    p.add_argument('--gt_file', type=str, default=None)
    p.add_argument('--test_gt_file', type=str, default=None)
    p.add_argument('--filenames_file', type=str, default=os.path.join(d, 'train_real.txt'))
    p.add_argument('--test_filenames_file', type=str, default=None)
    p.add_argument('--visual', type=str2bool, default='false', help='Visualize obtained images to debug (not built)')
    p.add_argument('--save_visual', type=str2bool, default='True', help='Save images for report')
    p.add_argument('--artifact_mode', type=str, default='None', help='Add aftifacts to the images (not built)', choices=['noise', 'None'])
    p.add_argument('--img_w', type=int, default=WIDTH)
    p.add_argument('--img_h', type=int, default=HEIGHT)
    p.add_argument('--full_img_w', type=int, default=FULL_WIDTH)
    p.add_argument('--full_img_h', type=int, default=FULL_HEIGHT)
    p.add_argument('--patch_size', type=int, default=PATCH_SIZE)
    p.add_argument('--batch_size', type=int, default=128)
    p.add_argument('--max_epoches', type=int, default=1)
    p.add_argument('--num_features', type=int, default=8, help='Number of features used to do RANSAC')
    p.add_argument('--num_iterations', type=int, default=100, help='Number of iterations used to do direct method')
    p.add_argument('--resume', type=str2bool, default='False', help='True: restore the existing model. False: retrain')
    # new
    p.add_argument('--synthetic', type=int, default=0, help='generate this many full-size pairs on the device instead of reading data_path')
    p.add_argument('--seed', type=int, default=0)
    return p


def resolve_paths(args):
    """The test files under --data_path (the reference's TEST_* defaults, :40-45) and the log / results dirs (:100-107)."""
    d = args.data_path
    args.test_pts1_file = args.test_pts1_file or os.path.join(d, 'test_pts1.txt')
    args.test_filenames_file = args.test_filenames_file or os.path.join(d, 'test_real.txt')
    args.test_gt_file = args.test_gt_file or os.path.join(d, 'test_gt.txt')
    prefix = args.method + '/'
    for a in args.augment_list:
        prefix += '_' + a
    prefix += '/' + 'RHO_' + str(RHO) + '_maxfeat_' + str(args.num_features) + '_doaugment_' + str(args.do_augment) + '/'
    args.log_dir = os.path.join(args.log_dir, prefix + args.mode + '/')
    args.results_dir = os.path.join(args.results_dir, prefix + args.mode + '/')
    return args


def find_percentile(values):
    """utils/utils.py:655-673: [mean, std] of the sorted list's 0-30 %, 30-60 % and 60-100 % parts."""
    v = np.sort(np.asarray(values, np.float64))
    out, start = [], 0
    for i, top in enumerate([0.3, 0.6, 1]):
        print('>> Top %.0f -  %.0f %%' % ([0.3, 0.6, 1][i - 1] * 100 if i >= 1 else 0, top * 100))
        stop = int(top * len(v))
        part = v[start:stop]
        out.append([float(np.mean(part)) if len(part) else float('nan'), float(np.std(part)) if len(part) else float('nan')])
        start = stop
    return out


def summarise(h_losses, num_fail, total_time, num_samples):
    """The five numbers of results.txt (:264): samples, mean h_loss, std, failure fraction, seconds per sample."""
    h = np.asarray(h_losses, np.float64)
    return [num_samples, float(np.mean(h)), float(np.std(h)), num_fail * 1.0 / num_samples, total_time / num_samples]


def write_pickle(args, h_losses):
    """h_losses.pkl under results_dir: the reference's dict (:248-256), as a Python 3 pickle of plain floats."""
    result = {'method': args.method, 'h_losses': [float(h) for h in h_losses], 'h_loss_mu': float(np.mean(h_losses)),
              'h_loss_std': float(np.std(h_losses))}
    path = os.path.join(args.results_dir, 'h_losses.pkl')
    with open(path, 'wb') as f:
        pickle.dump(result, f)
        print('===> Successfully write results  to  %s' % path)


def write_results_txt(args, line):
    """results.txt under log_dir: the five numbers of one line, '%.5f' (:265-267)."""
    path = os.path.join(args.log_dir, 'results.txt')
    with open(path, 'w') as f:
        np.savetxt(f, [line], delimiter=' ', fmt='%.5f')
        print('===> Wrote results to file %s' % path)


def run_batch(method, batch, num_iterations):
    """-> (h_loss [B] float64, fail [B] int, GPU seconds, pred_h4p [B,8] float32 clamped to +-80) for one extended
    Dataloader batch."""
    import torch
    from unsuperviseddeephomographyral2018_b200 import ops
    gt = torch.from_numpy(np.ascontiguousarray(batch["gt_corr"], np.float32)).cuda()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if method == 'direct':
        g1, g2 = ops.ecc_prep_u8(batch["I_u8"], batch["I_prime_u8"], batch.get("aug"))
        W, _, _, status = ops.find_homography_ecc(g1, g2, None, num_iterations, 1e-10)
    else:                                                             # identity: W = I, never "not found"
        B = gt.shape[0]
        W = torch.eye(3, device=gt.device).repeat(B, 1, 1).contiguous()
        status = torch.zeros(B, device=gt.device, dtype=torch.int32)
    pred, h, fail = ops.ecc_corr_h4p(W, status, gt)
    e1.record()
    torch.cuda.synchronize()
    return h.cpu().numpy(), fail.cpu().numpy(), e0.elapsed_time(e1) * 1e-3, pred.cpu().numpy()


def make_loader(args, batch_size):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    if args.synthetic:                                                # full-size pairs: the network size is the full size
        h, w = args.full_img_h, args.full_img_w
    else:
        h, w = args.img_h, args.img_w
    prm = dl.extended_dataloader_params(data_path=args.data_path, filenames_file=args.test_filenames_file, pts1_file=args.test_pts1_file,
                                        gt_file=args.test_gt_file, mode='test', batch_size=batch_size, img_h=h, img_w=w,
                                        patch_size=args.patch_size, augment_list=args.augment_list, do_augment=args.do_augment,
                                        full_img_h=args.full_img_h, full_img_w=args.full_img_w)
    return dl.Dataloader(prm, shuffle=False, synthetic_pairs=args.synthetic, seed=args.seed, device="cuda", rho=RHO)


def test(args):
    from unsuperviseddeephomographyral2018_b200 import _lib
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, report
    _lib.require_device()
    print('Save mean, std values to ', args.log_dir)
    print('Save images to', args.results_dir)
    if not args.resume:
        shutil.rmtree(args.log_dir, ignore_errors=True)
    os.makedirs(args.log_dir, exist_ok=True)
    os.makedirs(args.results_dir, exist_ok=True)
    num_data = args.synthetic if args.synthetic else dl.count_text_lines(args.test_filenames_file)
    print('===> There are totally %d test files' % num_data)
    batch_size = int(min(num_data, args.batch_size))
    steps = args.max_epoches * int(np.ceil(num_data / batch_size))
    loader = make_loader(args, batch_size)
    h_losses, num_fail, total_time, num_samples = [], 0, 0.0, 0
    for step in range(steps):
        b = loader.next_batch()
        h, f, secs, pred = run_batch(args.method, b, args.num_iterations)
        total_time += secs
        for i in range(len(h)):
            num_samples += 1
            if f[i] == 1:
                print('===> Fail case 1: Not found homography')
            elif f[i] == 2:
                print('===> Fail case 2:  error > identity')
            num_fail += int(f[i] != 0)
            h_losses.append(float(h[i]))
        if args.save_visual:
            # :250-267: the same drawing inline, pred_corr2 = pred_h4p + corr1 (h_loss after the failure substitution)
            corr1, corr2 = report.clicked_points(b["gt_corr"])
            names = [report.conventional_name(step * args.batch_size + i, float(h[i])) for i in range(len(h))]
            report.write(report.render(b, range(len(h)), corr1, corr2, pred.reshape(-1, 4, 2) + corr1, prime_left=False), names,
                         args.results_dir)
        print(' Test| image %d, h_loss %.3f, h_loss_average %.3f, fail %d/%d, time %.4f (batched)'
              % (num_samples - 1, h_losses[-1], np.mean(h_losses), num_fail, num_samples, secs / len(h)), flush=True)
    line = summarise(h_losses, num_fail, total_time, num_samples)
    write_pickle(args, h_losses)
    print('==========================================================')
    print('===> H_loss:', line[1], '+/-', line[2])
    print('Running time:', line[4], '(batched: GPU time of a batch / batch size)')
    print('Failure %.3f' % line[3])
    print('output_line:', line)
    write_results_txt(args, line)
    tops = find_percentile(h_losses)
    print('===> Percentile Values: (20, 50, 80, 100):')
    print(tops)
    print('======> End! ====================================')
    return line


def main(argv=None):
    print('<==================== Loading raw data ===================>\n')
    args = resolve_paths(build_parser().parse_args(argv))
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
