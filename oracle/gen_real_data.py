"""Host restatement of the real-data generator's pixel work (test reference and timing baseline, not a CLI option).

HostBackend         cv2.imread, cv2.resize to both sizes, cv2.cvtColor(..., COLOR_RGB2GRAY) for gray files and
                    cv2.imencode (cv2.imwrite's bytes): unsuperviseddeephomographyral2018_b200.gen_real_data.generate with
                    it is the host generator the device generator is compared with.
reference_samples   a transcription of homographyGeneration / dataCollection's loop (draws, indices, labels, cutoffs).
"""
import glob
import os
import random

import numpy as np


class HostBackend:
    def __init__(self, quality=95):
        self.quality = quality

    def frames(self, paths, size, full_size, gray):
        import cv2
        enc = lambda im: cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, self.quality])[1].tobytes()
        out = []
        for p in paths:
            I = cv2.imread(p)
            if I is None:
                raise IOError("cannot read %s" % p)
            full_I = cv2.resize(I, (full_size[1], full_size[0]))
            I = cv2.resize(I, (size[1], size[0]))
            if gray:
                I, full_I = cv2.cvtColor(I, cv2.COLOR_RGB2GRAY), cv2.cvtColor(full_I, cv2.COLOR_RGB2GRAY)
            out.append((enc(I), enc(full_I)))
        return out


def reference_samples(raw_image_path, ignore_list, num_data, start_index, im_per_im, rho, patch_size, height, corr=None, seed=0,
                      width=190, debug=False):
    """homographyGeneration's loop, transcribed with the reference's names (Python 2 division written as //).
    corr: (all_corr1, all_corr2) in test mode.  -> (next index, [(index, I file, I' file, pts1 row, test_gt row or None)])."""
    rnd = random.Random(seed)
    image_files = glob.glob(os.path.join(raw_image_path, '*.JPG'))
    image_files.sort()
    out, index = [], start_index
    for num_files in range(len(image_files) - 1):
        I_file = image_files[num_files]
        I_prime_file = image_files[num_files + 1]
        I_img_id = int(I_file[len(I_file) - 8: len(I_file) - 4])
        if I_img_id in ignore_list:
            continue
        if corr is not None:
            corr1 = corr[0][num_files * 4:num_files * 4 + 4].reshape([4, 2])
            corr2 = corr[1][num_files * 4:num_files * 4 + 4].reshape([4, 2])
        for i in range(im_per_im):
            x = rnd.randint(rho, width - rho - patch_size)
            y = (height - patch_size) // 2
            top_left_point = (x, y)
            bottom_left_point = (patch_size + x, y)
            bottom_right_point = (patch_size + x, patch_size + y)
            top_right_point = (x, patch_size + y)
            four_points = [top_left_point, bottom_left_point, bottom_right_point, top_right_point]
            if debug:
                index += 1
                return index, out
            pts1 = np.array(four_points).flatten().astype(np.float32)
            gt = np.hstack([corr1.flatten(), corr2.flatten()]) if corr is not None else None
            out.append((index, I_file, I_prime_file, pts1, gt))
            index += 1
            if index >= num_data + start_index:
                break
        if index >= start_index + num_data:
            break
    return index, out
