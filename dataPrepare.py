#!/usr/bin/env python
"""The reference's dataPrepare.py: cut the training scenes `scene_%04d/col_high_%04d.png` out of the source videos, each
frame down-sampled by 2 (INTER_AREA) -- here on the GPU (tecogan_b200/data_prepare.py), byte for byte the same files.

Same flags and defaults as the reference (dataPrepare.py:10-23), its configuration print and its stdout tee to
<summary_dir>/logfile_%m%d%H%M.txt.  The videos are not downloaded: each is read from <disk_path>/<vimeo id>.<ext>, where
the reference's youtube-dl leaves it, and a missing file is skipped.  One flag is added: --threads, the number of videos
decoded at once.  Making the frames needs a CUDA device; --TEST does not.

--scene_threshold T (extension, absent from the flags unless given; 0 < T <= 100) replaces the reference's table by
one made from every video directly in --disk_path (.mp4 .m4v .mov .mkv .webm .avi .mpg .mpeg .ts, sorted by name): each
is decoded whole, its hard cuts are found on the GPU by `main.py --scene_threshold`'s rule on the halved frames, and
every shot yields the disjoint --duration-frame scenes that fit inside it.  The cuts and the table are printed, in the
reference's syntax; the scenes are then written as the table's are, each video read in sequence instead of seeking
(DESIGN.md section 4.14).  With --TEST the table is found and printed, and nothing is written but the log; that scan
needs a CUDA device.
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
    # Opt-in: absent from the flags unless given, so a run without it keeps the reference's flag set.  Read as text and
    # checked by main(), so that a malformed value raises ValueError as an out-of-range one does.
    parser.add_argument('--scene_threshold', default=argparse.SUPPRESS,
                        help='(extension) cut the scenes from every video in disk_path at hard cuts scoring >= T, '
                             '0 < T <= 100 (main.py --scene_threshold\'s rule; 10 is a starting point), instead of '
                             'the reference\'s table; with --TEST the table is found and printed and only the log is written, '
                             'which then needs a CUDA device')
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
    """Run the command; `videos` replaces the reference's table (data_prepare.VIDEOS) for tests.  A bad
    --scene_threshold, or --duration < 1 with it, raises ValueError before anything is made or opened."""
    from tecogan_b200 import data_prepare
    from tecogan_b200.summary import Tee
    flags = parse_flags(argv)
    scanned = hasattr(flags, 'scene_threshold')
    if scanned:
        from tecogan_b200.lib.dataloader import scene_threshold
        flags.scene_threshold = scene_threshold(flags.scene_threshold)
        if flags.duration < 1:
            raise ValueError('--scene_threshold needs --duration >= 1, got %d' % flags.duration)
    os.makedirs(flags.disk_path, exist_ok=True)
    os.makedirs(flags.summary_dir, exist_ok=True)
    tee = Tee(log_path(flags.summary_dir))
    sys.stdout = tee
    try:
        print_configuration_op(flags)
        sources = None
        if scanned:
            videos, sources = data_prepare.scan(flags.disk_path, flags.scene_threshold, flags.duration,
                                                threads=flags.threads)
        data_prepare.prepare(data_prepare.VIDEOS if videos is None else videos, flags.disk_path, flags.start_id,
                             flags.duration, save_frames=not flags.TEST, remove=flags.REMOVE, threads=flags.threads,
                             sources=sources)
    finally:
        sys.stdout = tee.terminal
        tee.close()


if __name__ == '__main__':
    main()
