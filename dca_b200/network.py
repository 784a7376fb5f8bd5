"""Host-side mirror of dca/network.py: the ``AE_types`` registry and autoencoder objects with
the reference's method surface (.build .save .load_weights .predict .write), backed by the CUDA
engine instead of Keras graphs.

Flagship types (SURVEY.md section 8, tcgen05 path): 'zinb-conddisp' (dca/network.py:366-421), 'zinb'
(:496-550), 'nb-conddisp' (:293-339), 'nb' (:249-291).  The other registry keys -- 'normal' (:143-156),
'poisson' (:233-246), 'nb-shared' (:341-363), 'zinb-shared' (:465-493), 'zinb-elempi' (:424-462),
'nb-fork' (:664-760), 'zinb-fork' (:553-661) -- are re-parameterisations of the heads around the same loss
kernel and run on the shape-general fp32 path of the engine (csrc/extra_types.cu).
"""
from __future__ import annotations

import contextlib
import os
import pickle
from typing import Optional

import numpy as np
import torch

from .device_data import _one_dataset
from .engine import DeviceEngine
from .io import write_text_matrix, write_text_matrix_device

PREDICT_BATCH = 4096      # rows per dca_predict call (Keras predict uses 32; result is identical)


def _out_name(name, gzip):
    """The file name of one output matrix: <name>.tsv, or <name>.tsv.gz with gzip."""
    return name + (".tsv.gz" if gzip else ".tsv")


def gene_block(n_cells, n_genes, n_heads, free_bytes, max_block_bytes=None):
    """Genes per block of write_predictions: the device holds n_cells x block float32 per gene-major head, within half
    of free_bytes (the rest is left to the batch buffers and the text writer) and within max_block_bytes (all heads
    together) when given; at least one gene, at most n_genes."""
    budget = free_bytes // 2
    if max_block_bytes is not None:
        budget = min(budget, int(max_block_bytes))
    per_gene = 4 * max(int(n_cells), 1) * max(int(n_heads), 1)
    return int(max(1, min(int(n_genes), budget // per_gene)))


class Autoencoder:
    ae_type: Optional[str] = None      # key understood by the engine; None => not accelerated

    def __init__(self,
                 input_size,
                 output_size=None,
                 hidden_size=(64, 32, 64),
                 l2_coef=0.,
                 l1_coef=0.,
                 l2_enc_coef=0.,
                 l1_enc_coef=0.,
                 ridge=0.,
                 hidden_dropout=0.,
                 input_dropout=0.,
                 batchnorm=True,
                 activation='relu',
                 init='glorot_uniform',
                 file_path=None,
                 debug=False,
                 x_dtype='float32',
                 gemm_path='auto',
                 sharedpi=False,
                 sync_bn=False):
        self.input_size = input_size
        self.output_size = output_size if output_size is not None else input_size
        self.hidden_size = list(hidden_size)
        self.l2_coef, self.l1_coef = l2_coef, l1_coef
        self.l2_enc_coef, self.l1_enc_coef = l2_enc_coef, l1_enc_coef
        self.ridge = ridge
        self.hidden_dropout = hidden_dropout
        self.input_dropout = input_dropout
        self.batchnorm = batchnorm
        self.activation = activation
        self.init = init
        self.file_path = file_path
        self.debug = debug                 # train(): the loss kernels' inf/NaN checks of dca/loss.py:87-100 (train._DebugChecks)
        self.x_dtype = x_dtype
        self.gemm_path = gemm_path
        self.sharedpi = sharedpi           # ZINBAutoencoderElemPi only (dca/network.py:425-427)
        self.sync_bn = sync_bn             # multi-GPU: BatchNorm statistics over the global batch (no reference counterpart)
        self.loss = None
        self.extra_models = {}
        self.model = None          # the reference exposes a Keras model here; ours is .engine
        self.encoder = None
        self.engine: Optional[DeviceEngine] = None
        self._seed = 0

        if isinstance(self.hidden_dropout, list):
            assert len(self.hidden_dropout) == len(self.hidden_size)
        else:
            self.hidden_dropout = [self.hidden_dropout] * len(self.hidden_size)

    # -- dca/network.py:92-156
    def build(self, max_batch: int = 32, seed: Optional[int] = None):
        if self.ae_type is None:
            raise NotImplementedError("autoencoder type %s is not on the GPU-accelerated path"
                                      % type(self).__name__)
        if seed is not None:
            self._seed = seed
        self._max_batch = max_batch
        self.engine = DeviceEngine(self.input_size, self.output_size, self.hidden_size, self.ae_type,
                                   self.batchnorm, max_batch=max(max_batch, 1), x_dtype=self.x_dtype,
                                   ridge=self.ridge, l1=self.l1_coef, l2=self.l2_coef,
                                   l1_enc=self.l1_enc_coef, l2_enc=self.l2_enc_coef,
                                   gemm_path=self.gemm_path, seed=self._seed, sharedpi=self.sharedpi,
                                   sync_bn=self.sync_bn, activation=self.activation,
                                   hidden_dropout=self.hidden_dropout, input_dropout=self.input_dropout,
                                   init=self.init)
        self.model = self.engine
        self.encoder = self.engine
        self.loss = self.ae_type

    def ensure_engine(self, max_batch: int) -> DeviceEngine:
        """(Re)size the engine workspace for ``max_batch`` rows, keeping the weights."""
        if self.engine is None:
            self.build(max_batch=max_batch)
        elif self.engine.max_batch < max_batch:
            w = self.engine.get_weights()
            self.engine.close()
            self.build(max_batch=max_batch)
            self.engine.set_weights(w)
        return self.engine

    def summary(self) -> str:
        lines = ["%-28s %10s" % ("tensor", "shape")]
        for name, off, r, c in self.engine.param_info:
            lines.append("%-28s %10s" % (name, "(%d, %d)" % (r, c) if name.endswith("/kernel") else "(%d,)" % c))
        lines.append("total trainable parameters: %d" % self.engine.n_params)
        return "\n".join(lines)

    def penalty_value(self) -> float:
        """Kernel-regulariser term Keras adds to (val_)loss -- dca/network.py:125; 0 by default."""
        if not any((self.l1_coef, self.l2_coef, self.l1_enc_coef, self.l2_enc_coef)):
            return 0.0
        w = self.engine.get_weights()
        center = len(self.hidden_size) // 2
        tot = 0.0
        names = [n for n in w if n.endswith("/kernel")]
        for n in names:
            layer = n.split("/")[0]
            enc = layer == "center" or layer.startswith("enc")
            l1 = self.l1_enc_coef if (enc and self.l1_enc_coef != 0.) else self.l1_coef
            l2 = self.l2_enc_coef if (enc and self.l2_enc_coef != 0.) else self.l2_coef
            tot += l1 * np.abs(w[n]).sum() + l2 * np.square(w[n]).sum()
        return float(tot)

    # -- dca/network.py:158-167
    def save(self):
        if self.file_path:
            os.makedirs(self.file_path, exist_ok=True)
            with open(os.path.join(self.file_path, 'model.pickle'), 'wb') as f:
                pickle.dump(self, f)

    def __getstate__(self):
        st = dict(self.__dict__)
        for k in ("engine", "model", "encoder"):
            st[k] = None
        return st

    def save_weights(self, filename):
        """.npz with the reference's tensor names (h5py is not in the image; SURVEY.md section 5)."""
        np.savez(filename, **{k.replace("/", "__"): v for k, v in self.engine.get_weights().items()})

    def load_weights(self, filename):
        data = np.load(filename)
        if self.engine is None:
            self.build()
        self.engine.set_weights({k.replace("__", "/"): data[k] for k in data.files})
        self.encoder = self.engine

    # -- one fused inference pass instead of the reference's four Keras predict() calls
    def _run_predict(self, adata, want_mean, want_disp, want_pi, want_latent, device_data=None, stream_data=None,
                     packed_data=None):
        # a model without a dropout head has no pi: the engine writes nothing there, so none is returned (not the
        # uninitialised contents of the output buffer)
        want_pi = want_pi and self.has_pi
        eng, N, bs, run, theta, session = self._source(adata, _one_dataset(device_data, stream_data, packed_data))
        with session():
            return self._predict_batches(eng, N, bs, want_mean, want_disp, want_pi, want_latent, run, theta)

    # -- the input of the batched inference: (engine, cells, batch rows, run, theta, session) as
    # device_data._Dataset._predictor describes them, from a dataset or else from adata (X and obs['size_factors'])
    def _source(self, adata, data):
        if data is None:
            if adata is None:
                raise ValueError("give adata, device_data, stream_data or packed_data")
            return self._host_source(adata)
        data._cover(adata)
        eng = self.ensure_engine(max_batch=max(getattr(self, "_max_batch", 32), min(PREDICT_BATCH, data.n)))
        data._bind(eng)
        bs = min(PREDICT_BATCH, eng.max_batch)
        return (eng, data.n, bs) + data._predictor(eng, bs)

    def _host_source(self, adata):
        X = np.ascontiguousarray(np.asarray(adata.X), dtype=np.float32)
        eng = self.ensure_engine(max_batch=max(getattr(self, "_max_batch", 32), min(PREDICT_BATCH, X.shape[0])))
        dev = eng.device
        sf = np.asarray(adata.obs['size_factors'], dtype=np.float32).reshape(-1)

        def run(i, s, e, b):
            xd = torch.from_numpy(X[s:e]).to(dev).to(eng.x_dtype)
            sd = torch.from_numpy(sf[s:e]).to(dev)
            eng.predict(xd, sd, mean=b.get("mean"), disp=b.get("disp"), pi=b.get("pi"), latent=b.get("latent"))

        def theta(th):
            xd = torch.from_numpy(X[:1]).to(dev).to(eng.x_dtype)
            sd = torch.from_numpy(sf[:1]).to(dev)
            eng.predict(xd, sd, disp=th)
        return eng, X.shape[0], min(PREDICT_BATCH, eng.max_batch), run, theta, contextlib.nullcontext

    def _predict_batches(self, eng, N, bs, want_mean, want_disp, want_pi, want_latent, run, theta):
        """The outputs of run(i, s, e, buffers) -- the inference of batch i, rows [s, e), into one of two device buffer
        sets -- gathered on the host: each batch's outputs are copied to pinned host memory on a side stream, so the
        copy of one batch overlaps the next batch.  theta(th) writes the per-gene dispersion of the const-disp types."""
        dev = eng.device
        G = self.output_size
        cond = self.ae_type not in ("zinb", "nb", "poisson", "normal")
        Gs = 1 if self.ae_type in ("nb-shared", "zinb-shared") else G
        widths = {}
        if want_mean: widths["mean"] = G
        if want_disp and cond: widths["disp"] = Gs
        if want_pi: widths["pi"] = Gs
        if want_latent: widths["latent"] = eng.latent_dim
        out = {k: np.empty((N, w), np.float32) for k, w in widths.items()}
        bufs = [{k: torch.empty((bs, w), dtype=torch.float32, device=dev) for k, w in widths.items()} for _ in range(2)]
        pins = [{k: torch.empty((bs, w), dtype=torch.float32, pin_memory=True) for k, w in widths.items()} for _ in range(2)]
        pending = [None, None]
        comp = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)

        def drain(slot):
            ev, s, e = pending[slot]
            ev.synchronize()
            for k in widths:
                out[k][s:e] = pins[slot][k][: e - s].numpy()
            pending[slot] = None

        for i, s in enumerate(range(0, N, bs)):
            e, slot = min(s + bs, N), i % 2
            if pending[slot] is not None:
                drain(slot)                  # its copy has finished: the device buffers of this slot are free again
            b = bufs[slot]
            run(i, s, e, b)
            done = torch.cuda.Event()
            done.record(comp)
            side.wait_event(done)
            with torch.cuda.stream(side):
                for k in widths:
                    pins[slot][k][: e - s].copy_(b[k][: e - s], non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(side)
            pending[slot] = (copied, s, e)
        for slot in (0, 1):
            if pending[slot] is not None:
                drain(slot)
        res = {"mean": out.get("mean"), "pi": out.get("pi"), "latent": out.get("latent")}
        if want_disp:
            if cond:
                res["dispersion"] = out["disp"]
            else:
                th = torch.empty(G, dtype=torch.float32, device=dev)
                theta(th)
                res["dispersion"] = th.cpu().numpy()
        return res

    # -- dca/network.py:188-211
    def predict(self, adata, mode='denoise', return_info=False, copy=False, device_data=None, stream_data=None,
                packed_data=None):
        """device_data: a device_data.DeviceDataset of adata's cells; the input X and size factors are then read from
        it instead of adata.X / obs['size_factors'].  stream_data: a stream_data.StreamedDataset of adata's cells; the
        input batches are then streamed from its packed counts (the same outputs as from the DeviceDataset).
        packed_data: a packed_data.PackedDeviceDataset of adata's cells; the input batches are then expanded from its
        packed counts in device memory (the same outputs again)."""
        assert mode in ('denoise', 'latent', 'full'), 'Unknown mode'
        adata = adata.copy() if copy else adata
        res = self._run_predict(adata, mode in ('denoise', 'full'), False, False, mode in ('latent', 'full'), device_data,
                                stream_data, packed_data)
        if mode in ('latent', 'full'):
            print('dca: Calculating low dimensional representations...')
            adata.obsm['X_dca'] = res["latent"]
        if mode in ('denoise', 'full'):
            print('dca: Calculating reconstructions...')
            adata.X = res["mean"]
        if mode == 'latent':
            adata.X = adata.raw.X.copy()  # as the reference does (dca/network.py:208-209)
        return adata if copy else None

    def _device(self):
        """The engine's CUDA device (the current one before the engine exists): where write(gzip=True) compresses."""
        return self.engine.device if self.engine is not None else None

    # -- dca/network.py:213-231
    def write(self, adata, file_path, mode='denoise', colnames=None, gzip=False):
        """gzip=True writes each <name>.tsv as <name>.tsv.gz, compressed on the GPU (io.write_text_matrix)."""
        colnames = adata.var_names.values if colnames is None else colnames
        rownames = adata.obs_names.values
        print('dca: Saving output(s)...')
        os.makedirs(file_path, exist_ok=True)
        if mode in ('denoise', 'full'):
            print('dca: Saving denoised expression...')
            write_text_matrix(adata.X, os.path.join(file_path, _out_name('mean', gzip)),
                              rownames=rownames, colnames=colnames, transpose=True, gzip=gzip, device=self._device())
        if mode in ('latent', 'full'):
            print('dca: Saving latent representations...')
            write_text_matrix(adata.obsm['X_dca'], os.path.join(file_path, _out_name('latent', gzip)),
                              rownames=rownames, transpose=False, gzip=gzip, device=self._device())

    def write_predictions(self, file_path, rownames, colnames, mode='full', return_info=True, device_data=None,
                          stream_data=None, packed_data=None, adata=None, max_block_bytes=None, chunk_bytes=0,
                          gzip=False):
        """The files predict(adata, mode, return_info, ...) followed by write(adata, file_path, mode, colnames) write,
        byte for byte and with the same messages, without the cells x genes outputs ever on the host.  rownames: the
        cell labels (adata.obs_names), colnames: the output gene labels.  The input comes from device_data,
        stream_data or packed_data as in predict, else from adata (X and obs['size_factors']).

        mean.tsv, dispersion.tsv and dropout.tsv hold one line per gene, so they are written in gene blocks: per block,
        one inference pass over all cells keeps the block's columns of each of these heads on the device (cells x block
        float32 each, sized from free device memory and capped by max_block_bytes for all heads together), and
        io.write_text_matrix_device appends the block's lines to each file.  Every pass runs the same batches as
        predict, so the values are the ones predict returns; a model whose outputs fit one block is run once.
        latent.tsv comes from the first pass; the per-gene dispersion of 'nb' / 'zinb' from the same call as in
        predict, written by write_text_matrix.  The per-cell dispersion and dropout of 'nb-shared' / 'zinb-shared'
        are not cells x genes: with return_info those models go through predict(adata, ...) and write(...) unchanged,
        which needs adata.  chunk_bytes: the pinned text pieces of the writer (0: 16 MB).

        gzip=True writes <name>.tsv.gz in place of each <name>.tsv: the text is compressed on the GPU before it leaves
        it (one gzip member per gene block), and decompresses to the bytes gzip=False writes."""
        assert mode in ('denoise', 'latent', 'full'), 'Unknown mode'
        info = return_info and isinstance(self, _InfoMixin)
        if info and self.ae_type in ("nb-shared", "zinb-shared"):
            if adata is None:
                raise ValueError("%s writes its per-cell dispersion and dropout through predict and write: give adata"
                                 % self.ae_type)
            self.predict(adata, mode=mode, return_info=return_info, device_data=device_data, stream_data=stream_data,
                         packed_data=packed_data)
            self.write(adata, file_path, mode=mode, colnames=colnames, gzip=gzip)
            return
        eng, N, bs, run, theta, session = self._source(adata, _one_dataset(device_data, stream_data, packed_data))
        rownames, colnames = list(rownames), list(colnames)
        G = self.output_size
        if len(rownames) != N or len(colnames) != G:
            raise ValueError("got %d row and %d column labels for %d cells and %d output genes"
                             % (len(rownames), len(colnames), N, G))
        dev = eng.device
        cond = self.ae_type not in ("zinb", "nb", "poisson", "normal")
        want_mean, want_latent = mode in ('denoise', 'full'), mode in ('latent', 'full')
        want_pi = info and self.has_pi
        # the heads predict asks the engine for, and the gene-major ones written block by block
        widths = {}
        if want_mean: widths["mean"] = G
        if info and cond: widths["disp"] = G
        if want_pi: widths["pi"] = G
        if want_latent: widths["latent"] = eng.latent_dim
        files = [(k, _out_name(f, gzip)) for k, f in (("mean", "mean"), ("disp", "dispersion"), ("pi", "dropout"))
                 if k in widths]
        bufs = {k: torch.empty((bs, w), dtype=torch.float32, device=dev) for k, w in widths.items()}
        free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        block = gene_block(N, G, len(files), free, max_block_bytes)
        blk = {k: torch.empty((N, block), dtype=torch.float32, device=dev) for k, _ in files}
        latent = torch.empty((N, eng.latent_dim), dtype=torch.float32, device=dev) if want_latent else None

        if want_latent:
            print('dca: Calculating low dimensional representations...')
        if want_mean:
            print('dca: Calculating reconstructions...')
        print('dca: Saving output(s)...')
        os.makedirs(file_path, exist_ok=True)
        if want_mean:
            print('dca: Saving denoised expression...')
        for b, g0 in enumerate(range(0, G, block) if files else [0]):
            g1 = min(G, g0 + block)
            with session():
                for i, s in enumerate(range(0, N, bs)):
                    e = min(s + bs, N)
                    run(i, s, e, bufs)
                    for k, _ in files:
                        blk[k][s:e, :g1 - g0].copy_(bufs[k][:e - s, g0:g1])
                    if latent is not None and b == 0:
                        latent[s:e].copy_(bufs["latent"][:e - s])
            for k, f in files:
                # mean.tsv starts with the header of cell labels; dispersion.tsv and dropout.tsv have none
                write_text_matrix_device(blk[k][:, :g1 - g0], os.path.join(file_path, f),
                                         rownames=rownames if (k == "mean" and b == 0) else None,
                                         colnames=colnames[g0:g1], transpose=True, append=b > 0,
                                         chunk_bytes=chunk_bytes, gzip=gzip)
        del blk, bufs
        if want_latent:
            print('dca: Saving latent representations...')
            write_text_matrix_device(latent, os.path.join(file_path, _out_name('latent', gzip)), rownames=rownames,
                                     chunk_bytes=chunk_bytes, gzip=gzip)
        if info and not cond:
            th = torch.empty(G, dtype=torch.float32, device=dev)
            with session():
                theta(th)
            write_text_matrix(th.cpu().numpy().reshape(1, -1), os.path.join(file_path, _out_name('dispersion', gzip)),
                              colnames=colnames, transpose=True, gzip=gzip, device=dev)


class _InfoMixin:
    """Shared predict/write for the types that expose dispersion / dropout (dca/network.py:271-291,
    318-339, 395-421, 524-550): extra outputs are computed in the same fused inference pass."""
    has_pi = False
    const_disp = False

    def predict(self, adata, mode='denoise', return_info=False, copy=False, colnames=None, device_data=None,
                stream_data=None, packed_data=None):
        assert mode in ('denoise', 'latent', 'full'), 'Unknown mode'
        adata = adata.copy() if copy else adata
        res = self._run_predict(adata, mode in ('denoise', 'full'), return_info, return_info and self.has_pi,
                                mode in ('latent', 'full'), device_data, stream_data, packed_data)
        if return_info:
            if self.const_disp:
                adata.var['X_dca_dispersion'] = res["dispersion"]
            else:
                adata.obsm['X_dca_dispersion'] = res["dispersion"]
            if self.has_pi:
                adata.obsm['X_dca_dropout'] = res["pi"]
        if mode in ('latent', 'full'):
            print('dca: Calculating low dimensional representations...')
            adata.obsm['X_dca'] = res["latent"]
        if mode in ('denoise', 'full'):
            print('dca: Calculating reconstructions...')
            adata.X = res["mean"]
        if mode == 'latent':
            adata.X = adata.raw.X.copy()
        return adata if copy else None

    def write(self, adata, file_path, mode='denoise', colnames=None, gzip=False):
        colnames = adata.var_names.values if colnames is None else colnames
        Autoencoder.write(self, adata, file_path, mode, colnames=colnames, gzip=gzip)
        z = dict(gzip=gzip, device=self._device())
        if self.const_disp:
            if 'X_dca_dispersion' in adata.var_keys():
                write_text_matrix(np.asarray(adata.var['X_dca_dispersion']).reshape(1, -1),
                                  os.path.join(file_path, _out_name('dispersion', gzip)), colnames=colnames,
                                  transpose=True, **z)
        elif 'X_dca_dispersion' in adata.obsm_keys():
            write_text_matrix(adata.obsm['X_dca_dispersion'], os.path.join(file_path, _out_name('dispersion', gzip)),
                              colnames=colnames, transpose=True, **z)
        if 'X_dca_dropout' in adata.obsm_keys():
            write_text_matrix(adata.obsm['X_dca_dropout'], os.path.join(file_path, _out_name('dropout', gzip)),
                              colnames=colnames, transpose=True, **z)


class NBConstantDispAutoencoder(_InfoMixin, Autoencoder):     # 'nb'
    ae_type = "nb"; const_disp = True


class NBAutoencoder(_InfoMixin, Autoencoder):                 # 'nb-conddisp'
    ae_type = "nb-conddisp"


class ZINBAutoencoder(_InfoMixin, Autoencoder):               # 'zinb-conddisp'
    ae_type = "zinb-conddisp"; has_pi = True


class ZINBConstantDispAutoencoder(_InfoMixin, Autoencoder):   # 'zinb'
    ae_type = "zinb"; has_pi = True; const_disp = True


class PoissonAutoencoder(Autoencoder):                        # 'poisson'  dca/network.py:233-246
    ae_type = "poisson"


class NormalAutoencoder(Autoencoder):                         # 'normal'   dca/network.py:143-156 (the base class there)
    ae_type = "normal"


class NBSharedAutoencoder(_InfoMixin, Autoencoder):           # 'nb-shared'   dca/network.py:341-363
    ae_type = "nb-shared"


class ZINBSharedAutoencoder(_InfoMixin, Autoencoder):         # 'zinb-shared' dca/network.py:465-493
    ae_type = "zinb-shared"; has_pi = True


class ZINBAutoencoderElemPi(_InfoMixin, Autoencoder):         # 'zinb-elempi' dca/network.py:424-462 (network_kwds sharedpi)
    ae_type = "zinb-elempi"; has_pi = True


class NBForkAutoencoder(_InfoMixin, Autoencoder):             # 'nb-fork'     dca/network.py:664-760
    ae_type = "nb-fork"


class ZINBForkAutoencoder(_InfoMixin, Autoencoder):           # 'zinb-fork'   dca/network.py:553-661
    ae_type = "zinb-fork"; has_pi = True


# same keys as dca/network.py:763-768
AE_types = {'normal': NormalAutoencoder, 'poisson': PoissonAutoencoder,
            'nb': NBConstantDispAutoencoder, 'nb-conddisp': NBAutoencoder,
            'nb-shared': NBSharedAutoencoder, 'nb-fork': NBForkAutoencoder,
            'zinb': ZINBConstantDispAutoencoder, 'zinb-conddisp': ZINBAutoencoder,
            'zinb-shared': ZINBSharedAutoencoder, 'zinb-fork': ZINBForkAutoencoder,
            'zinb-elempi': ZINBAutoencoderElemPi}
