"""python -m oracle_assemble: the oracle is pure numpy; this only builds the voxel-grid oracle it calls."""
import oracle_prep

print(oracle_prep.build(verbose=True))
