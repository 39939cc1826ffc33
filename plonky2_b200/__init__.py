"""plonky2_b200 -- H100-native (sm_90a CUDA) implementation of the plonky2 prover hot path:
Goldilocks NTT / coset-LDE, Poseidon Merkle commitment and the FRI commit phase, behind the C ABI in
include/plonky2_b200.h. This package is the host-side mirror of the reference's interface for that
path (same names, argument meaning and error behaviour); see DESIGN.md and INTEGRATION.md."""
from . import field  # noqa: F401
from ._native import (ConstraintError, ConstraintReport, Context, NativeError, ShapeError,  # noqa: F401
                      default_context)
from .challenger import Challenger  # noqa: F401
from .fft import (coset_fft, coset_fft_with_options, coset_ifft, fft, fft_with_options, ifft,  # noqa: F401
                  ifft_with_options, lde, lde_onto_coset)
from .fri import (FriBatchInfo, FriConfig, FriInstanceInfo, FriOracleInfo, FriParams,  # noqa: F401
                  FriPolynomialInfo, FriProof, prove_openings, standard_recursion_fri_config,
                  starky_standard_fast_fri_config)
from .hash import (MerkleCap, MerkleProof, MerkleTree, PoseidonHash, PoseidonPermutation,  # noqa: F401
                   verify_merkle_proof_to_cap)
from .polynomial_batch import SALT_SIZE, PolynomialBatch, random_field_elements_keyed  # noqa: F401
from .proof import OpeningSet, StarkOpeningSet, eval_commitments  # noqa: F401
from .stark import (FibonacciStark, Stark, StarkConfig, StarkProof, StarkProofWithPublicInputs,  # noqa: F401
                    commit_quotient_polys, compute_quotient_polys, eval_l_0_and_l_last, eval_vanishing_poly)
from .lookup import Column, Filter, GrandProductChallenge, Lookup, get_grand_product_challenge_set  # noqa: F401
from .cross_table_lookup import (CrossTableLookup, CtlCheckVars, CtlData, CtlZData, MultiStarkProof,  # noqa: F401
                                 TableWithColumns, check_ctls, prove_with_ctls)
from . import stark  # noqa: F401  (stark.prove: the starky prover, next to plonk.prove_with_witness)
from . import plonk  # noqa: F401  (plonk.compute_quotient_polys: the plonky2 circuit quotient)
from .batch_merkle_tree import (BatchMerkleTree, compress_merkle_proofs, decompress_merkle_proofs,  # noqa: F401
                                verify_batch_merkle_proof_to_cap)
from .batch_fri import BatchFriOracle, batch_prove_openings  # noqa: F401
