"""Generate the reference's synthetic dataset (code/utils/gen_synthetic_data.py, same flags and layout, plus --seed) with
the resize, warp and JPEG encode on the GPU.  See unsuperviseddeephomographyral2018_b200/gen_data.py.

    python gen_synthetic_data.py --mode train --raw_data_path coco/train2014/ --data_path data/synthetic/45/ --seed 0
    python gen_synthetic_data.py --mode test  --test_raw_data_path coco/val2014/ --data_path data/synthetic/45/ --seed 1
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from unsuperviseddeephomographyral2018_b200 import gen_data  # noqa: E402

if __name__ == "__main__":
    gen_data.main()
