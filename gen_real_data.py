"""Generate the reference's real-data set (code/utils/gen_real_data.py, same flags and layout, plus --seed and
--test_labels) from frame sequences, with the JPEG decode, resize and encode on the GPU.  See
unsuperviseddeephomographyral2018_b200/gen_real_data.py.

    python gen_real_data.py --mode train --raw_data_path frames/train/ --data_path data/real/24/ --seed 0
    python gen_real_data.py --mode test  --test_raw_data_path frames/test/ --data_path data/real/24/ --seed 1 \
        --test_labels frames/test/labels/*.mat
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from unsuperviseddeephomographyral2018_b200 import gen_real_data  # noqa: E402

if __name__ == "__main__":
    gen_real_data.main()
