"""Build an Oxford RobotCar root from the raw downloads (data/oxford/build_dataset.py's main(), one GPU, traversals in
turn):

    python scripts/build_oxford.py RAW LMS OUT --sdk DIR [--traversals T ...] [--batch 64] [--images]

RAW holds <t>/vo/vo.csv, <t>/stereo.timestamps, <t>/stereo/centre/<ts>.png and <t>/tags.csv; LMS holds
<t>/lms_front.timestamps and <t>/lms_front/<ts>.bin; DIR is the RobotCar SDK, of which only models/ and extrinsics/
are read.  Night traversals and those with OUT/<t>/tags.csv are skipped.  Images are not converted (INTEGRATION.md).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def positive(v):
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"must be a positive integer (got {v})")
    return n


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("raw", metavar="RAW")
    ap.add_argument("lms", metavar="LMS")
    ap.add_argument("out", metavar="OUT")
    ap.add_argument("--sdk", required=True, help="RobotCar SDK directory (models/, extrinsics/)")
    ap.add_argument("--traversals", nargs="+", default=None, help="only these traversals (default: all of RAW)")
    ap.add_argument("--batch", type=positive, default=64, help="clouds (and images) per device call")
    ap.add_argument("--images", action="store_true", help="also convert the stereo-centre PNGs to JPEG")
    a = ap.parse_args(argv)
    from deepi2p_b200 import oxford_build
    oxford_build.build_root(a.raw, a.lms, a.out, a.sdk, traversals=a.traversals, batch=a.batch,
                            images=a.images)


if __name__ == "__main__":
    main()
