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

import os
import pickle
from typing import Optional

import numpy as np
import torch

from .engine import DeviceEngine
from .io import write_text_matrix

PREDICT_BATCH = 4096      # rows per dca_predict call (Keras predict uses 32; result is identical)


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
        self.debug = debug
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
        if self.init != 'glorot_uniform':
            raise NotImplementedError("only init='glorot_uniform' is on the accelerated path")
        if seed is not None:
            self._seed = seed
        self._max_batch = max_batch
        self.engine = DeviceEngine(self.input_size, self.output_size, self.hidden_size, self.ae_type,
                                   self.batchnorm, max_batch=max(max_batch, 1), x_dtype=self.x_dtype,
                                   ridge=self.ridge, l1=self.l1_coef, l2=self.l2_coef,
                                   l1_enc=self.l1_enc_coef, l2_enc=self.l2_enc_coef,
                                   gemm_path=self.gemm_path, seed=self._seed, sharedpi=self.sharedpi,
                                   sync_bn=self.sync_bn, activation=self.activation,
                                   hidden_dropout=self.hidden_dropout, input_dropout=self.input_dropout)
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
    def _run_predict(self, adata, want_mean, want_disp, want_pi, want_latent):
        X = np.ascontiguousarray(np.asarray(adata.X), dtype=np.float32)
        eng = self.ensure_engine(max_batch=max(getattr(self, "_max_batch", 32), min(PREDICT_BATCH, X.shape[0])))
        dev = eng.device
        sf = np.asarray(adata.obs['size_factors'], dtype=np.float32).reshape(-1)
        N, G = X.shape[0], self.output_size
        bs = min(PREDICT_BATCH, eng.max_batch)
        cond = self.ae_type not in ("zinb", "nb", "poisson", "normal")     # a dispersion head (vs per-gene theta / none)
        Gs = 1 if self.ae_type in ("nb-shared", "zinb-shared") else G       # per-cell heads: Dense(1)
        out = {}
        if want_mean: out["mean"] = np.empty((N, G), np.float32)
        if want_disp: out["dispersion"] = np.empty((N, Gs), np.float32) if cond else None
        if want_pi: out["pi"] = np.empty((N, Gs), np.float32)
        if want_latent: out["latent"] = np.empty((N, eng.latent_dim), np.float32)
        mean_d = torch.empty((bs, G), dtype=torch.float32, device=dev) if want_mean else None
        disp_d = torch.empty((bs, Gs), dtype=torch.float32, device=dev) if (want_disp and cond) else None
        pi_d = torch.empty((bs, Gs), dtype=torch.float32, device=dev) if want_pi else None
        lat_d = torch.empty((bs, eng.latent_dim), dtype=torch.float32, device=dev) if want_latent else None
        for s in range(0, N, bs):
            e = min(s + bs, N)
            xd = torch.from_numpy(X[s:e]).to(dev).to(eng.x_dtype)
            sd = torch.from_numpy(sf[s:e]).to(dev)
            eng.predict(xd, sd, mean=mean_d, disp=disp_d, pi=pi_d, latent=lat_d)
            if want_mean: out["mean"][s:e] = mean_d[: e - s].cpu().numpy()
            if disp_d is not None: out["dispersion"][s:e] = disp_d[: e - s].cpu().numpy()
            if want_pi: out["pi"][s:e] = pi_d[: e - s].cpu().numpy()
            if want_latent: out["latent"][s:e] = lat_d[: e - s].cpu().numpy()
        if want_disp and not cond:
            th = torch.empty(G, dtype=torch.float32, device=dev)
            xd = torch.from_numpy(X[:1]).to(dev).to(eng.x_dtype)
            sd = torch.from_numpy(sf[:1]).to(dev)
            eng.predict(xd, sd, disp=th)
            out["dispersion"] = th.cpu().numpy()
        return out

    # -- dca/network.py:188-211
    def predict(self, adata, mode='denoise', return_info=False, copy=False):
        assert mode in ('denoise', 'latent', 'full'), 'Unknown mode'
        adata = adata.copy() if copy else adata
        res = self._run_predict(adata, mode in ('denoise', 'full'), False, False, mode in ('latent', 'full'))
        if mode in ('latent', 'full'):
            print('dca: Calculating low dimensional representations...')
            adata.obsm['X_dca'] = res["latent"]
        if mode in ('denoise', 'full'):
            print('dca: Calculating reconstructions...')
            adata.X = res["mean"]
        if mode == 'latent':
            adata.X = adata.raw.X.copy()  # as the reference does (dca/network.py:208-209)
        return adata if copy else None

    # -- dca/network.py:213-231
    def write(self, adata, file_path, mode='denoise', colnames=None):
        colnames = adata.var_names.values if colnames is None else colnames
        rownames = adata.obs_names.values
        print('dca: Saving output(s)...')
        os.makedirs(file_path, exist_ok=True)
        if mode in ('denoise', 'full'):
            print('dca: Saving denoised expression...')
            write_text_matrix(adata.X, os.path.join(file_path, 'mean.tsv'),
                              rownames=rownames, colnames=colnames, transpose=True)
        if mode in ('latent', 'full'):
            print('dca: Saving latent representations...')
            write_text_matrix(adata.obsm['X_dca'], os.path.join(file_path, 'latent.tsv'),
                              rownames=rownames, transpose=False)


class _InfoMixin:
    """Shared predict/write for the types that expose dispersion / dropout (dca/network.py:271-291,
    318-339, 395-421, 524-550): extra outputs are computed in the same fused inference pass."""
    has_pi = False
    const_disp = False

    def predict(self, adata, mode='denoise', return_info=False, copy=False, colnames=None):
        assert mode in ('denoise', 'latent', 'full'), 'Unknown mode'
        adata = adata.copy() if copy else adata
        res = self._run_predict(adata, mode in ('denoise', 'full'), return_info, return_info and self.has_pi,
                                mode in ('latent', 'full'))
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

    def write(self, adata, file_path, mode='denoise', colnames=None):
        colnames = adata.var_names.values if colnames is None else colnames
        Autoencoder.write(self, adata, file_path, mode, colnames=colnames)
        if self.const_disp:
            if 'X_dca_dispersion' in adata.var_keys():
                write_text_matrix(np.asarray(adata.var['X_dca_dispersion']).reshape(1, -1),
                                  os.path.join(file_path, 'dispersion.tsv'), colnames=colnames, transpose=True)
        elif 'X_dca_dispersion' in adata.obsm_keys():
            write_text_matrix(adata.obsm['X_dca_dispersion'], os.path.join(file_path, 'dispersion.tsv'),
                              colnames=colnames, transpose=True)
        if 'X_dca_dropout' in adata.obsm_keys():
            write_text_matrix(adata.obsm['X_dca_dropout'], os.path.join(file_path, 'dropout.tsv'),
                              colnames=colnames, transpose=True)


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
