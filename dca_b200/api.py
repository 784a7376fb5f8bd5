"""``dca()`` with the signature of dca/api.py:19-45, re-pointed at the H100 engine."""
from __future__ import annotations

import os
import random

import numpy as np
import torch

from .anndata_lite import is_anndata
from .io import read_dataset, normalize, filter_genes_mask
from .train import train
from .network import AE_types


def dca(adata, mode='denoise', ae_type='nb-conddisp', normalize_per_cell=True, scale=True, log1p=True,
        # network
        hidden_size=(64, 32, 64), hidden_dropout=0., batchnorm=True, activation='relu', init='glorot_uniform',
        network_kwds={},
        # training
        epochs=300, reduce_lr=10, early_stop=15, batch_size=32, optimizer='RMSprop', learning_rate=None,
        random_state=0, threads=None, verbose=False, training_kwds={},
        # outputs
        return_model=False, return_info=False, copy=False, check_counts=True):
    """Deep count autoencoder (DCA) API -- drop-in for ``dca.api.dca`` (dca/api.py:19-211).

    Parameters and return values are those of the reference (see its docstring,
    dca/api.py:46-144): ``mode`` 'denoise' overwrites ``adata.X`` with the denoised mean,
    'latent' adds ``adata.obsm['X_dca']``; ``return_info`` adds ``obsm['X_dca_dispersion']``
    (``var[...]`` for the constant-dispersion types), ``obsm['X_dca_dropout']`` (ZINB types) and
    ``uns['dca_loss_history']``; raw counts are kept in ``adata.raw``.  ``threads`` is accepted
    and ignored (the arithmetic runs on the GPU).  ``network_kwds`` additionally understands
    ``x_dtype`` ('float32' | 'bfloat16') and ``gemm_path`` ('auto' | 'generic' | 'tcgen05').
    """
    assert is_anndata(adata), 'adata must be an AnnData instance'
    assert mode in ('denoise', 'latent'), '%s is not a valid mode.' % mode

    # set seed for reproducibility                                         (dca/api.py:150-153)
    random.seed(random_state)
    np.random.seed(random_state)
    torch.manual_seed(random_state)
    os.environ['PYTHONHASHSEED'] = '0'

    # 'preprocess': 'host' (default) | 'device' -- normalise on the GPU and keep X there (device_data.py); popped here
    # like the other keywords train() does not take from the reference
    training_kwds = dict(training_kwds)
    preprocess = training_kwds.pop('preprocess', 'host')
    if preprocess not in ('host', 'device'):
        raise ValueError("training_kwds['preprocess'] must be 'host' or 'device', got %r" % (preprocess,))
    # with 'preprocess': 'device', 'stream': True trains out of core (stream_data.StreamedDataset: packed counts in host
    # memory, the same results as the resident dataset); 'auto' does so when the resident dataset would not fit
    # 'packed': True keeps the raw counts packed in device memory (packed_data.PackedDeviceDataset: several times the
    # cells of the resident dataset, the same results)
    packed = training_kwds.pop('packed', False)
    if packed and preprocess != 'device':
        raise ValueError("training_kwds['packed'] needs 'preprocess': 'device'")
    if packed and training_kwds.get('stream', False):
        raise ValueError("training_kwds 'packed' and 'stream' exclude each other: the counts stay packed in device or "
                         "in host memory")
    streamed = False
    if preprocess == 'device' and training_kwds.get('stream', False) in (True, 'auto'):
        streamed = training_kwds.pop('stream')

    # raw counts go to adata.raw; the input object is copied only when copy=True  (dca/api.py:156-160)
    adata = read_dataset(adata, transpose=False, test_split=False, copy=copy, check_counts=check_counts)

    ds = None
    x_dtype = network_kwds.get('x_dtype', 'float32')
    if preprocess == 'device':
        # the same steps on the device; adata.X keeps the raw counts until predict() overwrites it
        from .device_data import DeviceDataset, build_dataset
        from .io import apply_device_normalize
        if streamed == 'auto':
            dev = torch.device('cuda', torch.cuda.current_device())
            streamed = DeviceDataset.device_bytes(adata.X, x_dtype, normalize_per_cell) > torch.cuda.mem_get_info(dev)[0]
        ds = build_dataset(adata.X, None, x_dtype, stream=streamed, packed=packed, batch=batch_size,
                           size_factors=normalize_per_cell, logtrans_input=log1p, normalize_input=scale)
        assert (ds.input_gene_totals >= 1).all(), 'Please remove all-zero genes before using DCA.'
        apply_device_normalize(adata, ds, filter_min_counts=False, set_x=False)
    else:
        # all-zero genes are an error, as in the reference                    (dca/api.py:163-164)
        nonzero_genes, _ = filter_genes_mask(adata.X, min_counts=1)
        assert nonzero_genes.all(), 'Please remove all-zero genes before using DCA.'

        # no filtering here: cell and gene indices stay those of the caller    (dca/api.py:166-170)
        adata = normalize(adata, filter_min_counts=False, size_factors=normalize_per_cell, normalize_input=scale,
                          logtrans_input=log1p)

    net_args = dict(network_kwds, hidden_size=hidden_size, hidden_dropout=hidden_dropout, batchnorm=batchnorm,
                    activation=activation, init=init)
    net = AE_types[ae_type](input_size=adata.n_vars, output_size=adata.n_vars, **net_args)
    net.save()
    net.build(max_batch=batch_size, seed=random_state)

    fit_args = dict(training_kwds, epochs=epochs, reduce_lr=reduce_lr, early_stop=early_stop, batch_size=batch_size,
                    optimizer=optimizer, verbose=verbose, threads=threads, learning_rate=learning_rate)
    if ds is None:
        hist = train(adata[adata.obs.dca_split == 'train'], net, **fit_args)
        res = net.predict(adata, mode, return_info, copy)
    else:
        train_mask = np.asarray(adata.obs.dca_split == 'train')
        # no AnnData subset: train() reads everything from the dataset, and a subset would copy the raw counts
        hist = train(None, net, **{ds.kind: ds.take(train_mask)}, **fit_args)
        res = net.predict(adata, mode, return_info, copy, **{ds.kind: ds})
    adata = res if copy else adata

    if return_info:
        adata.uns['dca_loss_history'] = hist.history

    if return_model:
        return (adata, net) if copy else net
    else:
        return adata if copy else None
