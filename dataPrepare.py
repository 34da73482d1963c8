#!/usr/bin/env python
"""The reference's dataPrepare.py: cut the training scenes `scene_%04d/col_high_%04d.png` out of the source videos, each
frame down-sampled by 2 (INTER_AREA) -- here on the GPU (tecogan_b200/data_prepare.py), byte for byte the same files.

Same flags and defaults as the reference (dataPrepare.py:10-23), its configuration print and its stdout tee to
<summary_dir>/logfile_%m%d%H%M.txt.  The videos are not downloaded: each is read from <disk_path>/<vimeo id>.<ext>, where
the reference's youtube-dl leaves it, and a missing file is skipped.  One flag is added: --threads, the number of videos
decoded at once.  Making the frames needs a CUDA device; --TEST does not.
"""
import argparse
import datetime
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse_flags(argv=None):
    parser = argparse.ArgumentParser(description='Process parameters.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument('--start_id', default=2000, type=int, help='starting scene index')
    parser.add_argument('--duration', default=120, type=int, help='scene duration')
    parser.add_argument('--disk_path', default="/mnt/netdisk/data/video/",
                        help='the directory of the source videos <id>.<ext>, where the scene folders are written')
    parser.add_argument('--summary_dir', default="", help='the path to save the log')
    parser.add_argument('--REMOVE', action='store_true',
                        help='whether to remove the original video file after data preparation')
    parser.add_argument('--TEST', action='store_true',
                        help='verify the source videos, save information in log, write no frames')
    parser.add_argument('--threads', default=4, type=int, help='videos decoded at once (extension)')
    flags = parser.parse_args(argv)
    if flags.summary_dir == "":
        flags.summary_dir = os.path.join(flags.disk_path, "log/")
    return flags


def print_configuration_op(flags):
    print('[Configurations]:')
    for name, value in flags.__dict__.items():
        print('\t%s: %s' % (name, str(value)))
    print('End of configuration')


def log_path(summary_dir, now=None):
    """The log the reference tees stdout to: <summary_dir>/logfile_%m%d%H%M.txt, appended to."""
    now = now or datetime.datetime.now()
    return os.path.join(summary_dir, "logfile_%s.txt" % now.strftime("%m%d%H%M"))


def main(argv=None, videos=None):
    """Run the command; `videos` replaces the reference's table (data_prepare.VIDEOS) for tests."""
    from tecogan_b200 import data_prepare
    from tecogan_b200.summary import Tee
    flags = parse_flags(argv)
    os.makedirs(flags.disk_path, exist_ok=True)
    os.makedirs(flags.summary_dir, exist_ok=True)
    tee = Tee(log_path(flags.summary_dir))
    sys.stdout = tee
    try:
        print_configuration_op(flags)
        data_prepare.prepare(data_prepare.VIDEOS if videos is None else videos, flags.disk_path, flags.start_id,
                             flags.duration, save_frames=not flags.TEST, remove=flags.REMOVE, threads=flags.threads)
    finally:
        sys.stdout = tee.terminal
        tee.close()


if __name__ == '__main__':
    main()
