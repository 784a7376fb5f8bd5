"""Command line with the flags of dca/__main__.py:18-138 (``dca input outputdir [...]``)."""
import argparse

# (flags, kwargs) in the reference's order; paired --x/--nox booleans share a dest
_OPTIONS = [
    (('input',), dict(type=str, help='Input is raw count data in TSV/CSV, Matrix Market (.mtx), their .gz, or H5AD '
                                     '(anndata) format, or a Cell Ranger matrix directory (matrix.mtx[.gz], '
                                     'features.tsv[.gz] or genes.tsv[.gz], barcodes.tsv[.gz], with or without a GEO '
                                     'sample prefix: cells named by barcode, genes by unique gene symbol, Gene '
                                     'Expression rows only). Row/col names are mandatory. TSV/CSV and Matrix Market '
                                     'files and directories must be gene x cell (use -t for cell x gene); H5AD files '
                                     'must be cell x gene.')),
    (('outputdir',), dict(type=str, help='The path of the output directory')),
    (('--normtype',), dict(type=str, default='zheng', help='Type of size factor estimation (parsed, unused; default: zheng)')),
    (('-t', '--transpose'), dict(dest='transpose', action='store_true', help='Transpose input matrix (default: False)')),
    (('--testsplit',), dict(dest='testsplit', action='store_true', help='Use one fold as a test set (default: False)')),
    (('--type',), dict(type=str, default='nb-conddisp', help='Type of autoencoder. Accelerated: nb, nb-conddisp (default), '
                                                             'zinb, zinb-conddisp')),
    (('--threads',), dict(type=int, default=None, help='Accepted for compatibility; ignored on the GPU path')),
    (('-b', '--batchsize'), dict(type=int, default=32, help='Batch size (default:32)')),
    (('--sizefactors',), dict(dest='sizefactors', action='store_true', help='Normalize means by library size (default: True)')),
    (('--nosizefactors',), dict(dest='sizefactors', action='store_false', help='Do not normalize means by library size')),
    (('--norminput',), dict(dest='norminput', action='store_true', help='Zero-mean normalize input (default: True)')),
    (('--nonorminput',), dict(dest='norminput', action='store_false', help='Do not zero-mean normalize inputs')),
    (('--loginput',), dict(dest='loginput', action='store_true', help='Log-transform input (default: True)')),
    (('--nologinput',), dict(dest='loginput', action='store_false', help='Do not log-transform inputs')),
    (('-d', '--dropoutrate'), dict(type=str, default='0.0', help='Dropout rate (default: 0)')),
    (('--batchnorm',), dict(dest='batchnorm', action='store_true', help='Batchnorm (default: True)')),
    (('--nobatchnorm',), dict(dest='batchnorm', action='store_false', help='Do not use batchnorm')),
    (('--l2',), dict(type=float, default=0.0, help='L2 regularization coefficient (default: 0.0)')),
    (('--l1',), dict(type=float, default=0.0, help='L1 regularization coefficient (default: 0.0)')),
    (('--l2enc',), dict(type=float, default=0.0, help='Encoder-specific L2 regularization coefficient (default: 0.0)')),
    (('--l1enc',), dict(type=float, default=0.0, help='Encoder-specific L1 regularization coefficient (default: 0.0)')),
    (('--ridge',), dict(type=float, default=0.0, help='L2 regularization coefficient for dropout probabilities (default: 0.0)')),
    (('--gradclip',), dict(type=float, default=5.0, help='Clip grad values (default: 5.0)')),
    (('--activation',), dict(type=str, default='relu', help='Activation function of hidden units (default: relu)')),
    (('--optimizer',), dict(type=str, default='RMSprop', help='Optimization method (default: RMSprop)')),
    (('--init',), dict(type=str, default='glorot_uniform', help='Initialization method for weights (default: glorot_uniform)')),
    (('-e', '--epochs'), dict(type=int, default=300, help='Max number of epochs (default: 300)')),
    (('--earlystop',), dict(type=int, default=15, help='Epochs without val_loss improvement before stopping (default: 15)')),
    (('--reducelr',), dict(type=int, default=10, help='Epochs without val_loss improvement before lr*0.1 (default: 10)')),
    (('-s', '--hiddensize'), dict(type=str, default='64,32,64', help='Size of hidden layers (default: 64,32,64)')),
    (('--inputdropout',), dict(type=float, default=0.0, help='Input layer dropout probability')),
    (('-r', '--learningrate'), dict(type=float, default=None, help='Learning rate (default: 0.001)')),
    (('--saveweights',), dict(dest='saveweights', action='store_true', help='Save weights (default: False)')),
    (('--no-saveweights',), dict(dest='saveweights', action='store_false', help='Do not save weights')),
    (('--hyper',), dict(dest='hyper', action='store_true', help='Hyperparameter search (not on the accelerated path)')),
    (('--hypern',), dict(dest='hypern', type=int, default=1000, help='(hyper) number of samples')),
    (('--hyperepoch',), dict(dest='hyperepoch', type=int, default=100, help='(hyper) epochs per sample')),
    (('--debug',), dict(dest='debug', action='store_true',
                        help='Check the NB/ZINB loss terms y_pred, t1 and t2 of every element for inf/NaN on the GPU in '
                             'every training and validation step and stop with FloatingPointError at the first batch '
                             'that has one, naming its cell and gene; no-op for the nb, poisson and normal types, as in '
                             'DCA (default: False)')),
    (('--tensorboard',), dict(dest='tensorboard', action='store_true', help='Not on the accelerated path')),
    (('--checkcounts',), dict(dest='checkcounts', action='store_true', help='Check that the matrix has raw counts (default: True)')),
    (('--nocheckcounts',), dict(dest='checkcounts', action='store_false', help='Do not check for raw counts')),
    (('--denoisesubset',), dict(dest='denoisesubset', type=str, help='Denoise only the genes listed (one per line) in this file')),
    (('--preprocess',), dict(type=str, default='host', choices=('host', 'device'),
                             help='Where size factors, log1p and scaling are computed: host (NumPy, default) or device '
                                  '(on the GPU; the normalised matrix then stays in GPU memory for training and prediction)')),
    (('--stream',), dict(dest='stream', action='store_true',
                         help='With --preprocess device: keep the raw counts packed in host memory and stream them '
                              'through the GPU for preprocessing, training and prediction (data larger than GPU memory; '
                              'same results)')),
    (('--packed',), dict(dest='packed', action='store_true',
                         help='With --preprocess device: keep the raw counts packed in GPU memory (several times more '
                              'cells than the normalised matrix; every batch is expanded on the GPU; same results)')),
    (('--gzip',), dict(dest='gzip', action='store_true',
                       help='Write the output matrices gzip-compressed (mean.tsv.gz, ...; compressed on the GPU)')),
]

_DEFAULTS = dict(transpose=False, testsplit=False, saveweights=False, sizefactors=True, batchnorm=True,
                 checkcounts=True, norminput=True, hyper=False, debug=False, tensorboard=False, loginput=True,
                 stream=False, packed=False, gzip=False)


def build_parser():
    parser = argparse.ArgumentParser(prog='dca', description='Autoencoder (H100-native DCA hot path)')
    for flags, kw in _OPTIONS:
        parser.add_argument(*flags, **kw)
    parser.set_defaults(**_DEFAULTS)
    return parser


def parse_args(argv=None):
    return build_parser().parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    # import the engine only after parse_args() so that --help stays fast (as the reference does)
    from . import train
    train.train_with_args(args)


if __name__ == '__main__':
    main()
