"""Build tests/golden/biochemists.npz from the reference's own R-fitted fixtures.

Needs a checkout of theislab/dca:  python tests/golden/make_golden.py /path/to/dca-checkout

Sources (theislab/dca @ 6abd124, read-only data files, provenance data/biochemists.R:16-42):
  data/biochemists.tsv                   915 x 6 table: count response `art` + 5 covariates
  data/biochemists-nb-coef.tsv           MASS::glm.nb coefficients + theta
  data/biochemists-nb-predictions.tsv    fitted NB means
  data/biochemists-zinb-coef.tsv         pscl::zeroinfl(dist="negbin") count/zero coefficients + theta
  data/biochemists-zinb-predictions.tsv  fitted (zero prob, count mean)

The .npz carries the numeric content of those tables plus two known-answer values
computed here with the float64 oracle (summed NLL at R's MLE); tests assert the
oracle reproduces R's fitted values (pins mu/pi parametrisation) and that the
gradient of the oracle's NLL vanishes at R's MLE (pins the loss formulas of
dca/loss.py:87-88,130-138).
"""
import os, sys
import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import dca_oracle as O  # noqa: E402


def main():
    REF = os.path.join(sys.argv[1], "data")
    tab = pd.read_csv(os.path.join(REF, "biochemists.tsv"), sep="\t")
    y = tab["art"].to_numpy(np.float64)
    cov = tab[["fem", "mar", "kid5", "phd", "ment"]].to_numpy(np.float64)
    design = np.concatenate([np.ones((len(y), 1)), cov], axis=1)
    nb = pd.read_csv(os.path.join(REF, "biochemists-nb-coef.tsv"), sep="\t")
    zi = pd.read_csv(os.path.join(REF, "biochemists-zinb-coef.tsv"), sep="\t")
    nb_pred = pd.read_csv(os.path.join(REF, "biochemists-nb-predictions.tsv"), sep="\t")["count"].to_numpy()
    zi_pred = pd.read_csv(os.path.join(REF, "biochemists-zinb-predictions.tsv"), sep="\t")
    nb_beta = nb["val"].to_numpy()[:6]; nb_theta = float(nb["val"].to_numpy()[6])
    zi_count = zi["count"].to_numpy()[:6]; zi_zero = zi["zero"].to_numpy()[:6]
    zi_theta = float(zi["count"].to_numpy()[6])

    mu_nb = np.exp(design @ nb_beta)
    kat_nb = float(np.sum(O.nb_loss_elem(y, mu_nb, np.full_like(y, nb_theta))))
    mu_zi = np.exp(design @ zi_count)
    pi_zi = 1.0 / (1.0 + np.exp(-(design @ zi_zero)))
    kat_zinb = float(np.sum(O.zinb_loss_elem(y, mu_zi, np.full_like(y, zi_theta), pi_zi)))
    print("KAT nb  sum NLL  =", repr(kat_nb))
    print("KAT zinb sum NLL =", repr(kat_zinb))
    np.savez_compressed(os.path.join(HERE, "biochemists.npz"),
                        y=y, design=design, nb_beta=nb_beta, nb_theta=nb_theta, nb_pred=nb_pred,
                        zinb_count=zi_count, zinb_zero=zi_zero, zinb_theta=zi_theta,
                        zinb_pred_zero=zi_pred["zero"].to_numpy(), zinb_pred_count=zi_pred["count"].to_numpy(),
                        kat_nb_sum_nll=kat_nb, kat_zinb_sum_nll=kat_zinb)


if __name__ == "__main__":
    main()
