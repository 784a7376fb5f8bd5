"""Drop-in alias: ``import dca`` resolves to the H100-native implementation (package dca_b200),
so callers of the reference's ``dca.api.dca`` / ``python -m dca`` need no change."""
