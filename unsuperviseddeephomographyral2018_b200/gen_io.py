"""What the two dataset generators (gen_data.py, gen_real_data.py) share: the reference's dataCollection deletions and
directories, and a background file writer."""
import os
import queue
import shutil
import threading


def prepare(args, dirs):
    """dataCollection's deletions (the same in both reference generators), then makedirs of `dirs` (None entries skipped).
    --resume N in train mode removes gt_file first: when it does not exist, the try-block stops there and nothing else is
    deleted."""
    if args.resume in ("N", "n") and args.start_index == 0 and args.mode == "train" and not args.debug:
        try:
            os.remove(args.gt_file)
            os.remove(args.pts1_file)
            os.remove(args.filenames_file)
            shutil.rmtree(args.I_dir, ignore_errors=True)
            if args.I_prime_dir is not None:
                shutil.rmtree(args.I_prime_dir, ignore_errors=True)
        except OSError:
            pass
    if args.resume in ("N", "n") and args.mode == "test" and not args.debug:
        try:
            os.remove(args.test_gt_file)
            os.remove(args.test_pts1_file)
            os.remove(args.test_filenames_file)
        except OSError:
            pass
    if not args.debug:
        for d in dirs:
            if d is not None:
                os.makedirs(d, exist_ok=True)


class Writer:
    """Writes (path, bytes) on a background thread; close() waits for every file and re-raises a write error."""

    def __init__(self):
        self.q, self.err = queue.Queue(maxsize=4096), None
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()

    def _run(self):
        while True:
            item = self.q.get()
            if item is None:
                return
            try:
                with open(item[0], "wb") as f:
                    f.write(item[1])
            except OSError as e:
                self.err = self.err or e

    def put(self, path, data):
        self.q.put((path, data))

    def close(self):
        self.q.put(None)
        self.t.join()
        if self.err:
            raise self.err
