"""Flag surface of the reference's options/options_test.py:20-76 for `python -m dvd_b200.test`, kept name for name, plus the
dataset's and the model's own flags (two-pass parse). `--html_logger` and `--manual_seed` are accepted; the HTML page and the
videos of the reference's `on_test_end` are not produced."""
import argparse
import sys


def add_general_arguments(parser):
    a = parser.add_argument
    a('--gpu', type=str, required=True, help="gpu idx ('-1' is rejected: dvd_b200 has no CPU path)")
    a('--dataset', type=str, required=True, help='name of the dataset')
    a('--workers', type=int, default=4, help='number of data loading workers')
    a('--batch_size', type=int, default=16, help='frames per test batch')
    a('--net', type=str, required=True, help='name of the model')
    a('--checkpoint_path', type=str, required=True, help='training log directory holding opt.pt, best.pt and nets/')
    a('--epoch', type=int, default=-1, help='epoch to test: nets/%%04d.pt, or best.pt when negative')
    a('--output_dir', type=str, required=True, help='output directory (prefix of <net>_<dataset>_<suffix>)')
    a('--overwrite', action='store_true', help='whether to overwrite the output folder if it exists')
    a('--suffix', default='epoch_{epoch}', type=str, help="suffix formatted with the options, e.g. '{classes}_lr{lr}'")
    a('--html_logger', action='store_true', help='accepted, no effect')
    a('--manual_seed', type=int, default=None, help='manual seed for randomness')
    return parser


def parse(argv=None, get_dataset=None, get_model=None):
    from ..models import get_model as _gm
    from ..datasets import get_dataset as _gd
    get_model, get_dataset = get_model or _gm, get_dataset or _gd
    argv = sys.argv[1:] if argv is None else argv
    parser = add_general_arguments(argparse.ArgumentParser())
    first, _ = parser.parse_known_args(argv)
    parser, _ = get_dataset(first.dataset).add_arguments(parser)
    parser, _ = get_model(first.net).add_arguments(parser)
    opt, unknown = parser.parse_known_args(argv)
    if unknown:
        print('[warning] ignoring unknown argument', unknown)
    return opt
