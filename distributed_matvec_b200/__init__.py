"""distributed_matvec_b200 -- matrix-free Hamiltonian-vector product on H100.

Host-side mirror of the reference's interface for the hot path (twesterhout/distributed-matvec,
src/DistributedMatrixVector.chpl + src/BatchedOperator.chpl); all compute is in libdmv_b200.so
(hand-written sm_90a CUDA behind the C ABI of include/dmv_b200.h).  No CPU fallback.
"""
from .config import BasisSpec, OperatorSpec, load_config_from_yaml  # noqa: F401
from .operator import (BatchedOperator, Basis, ChapelKernels, Operator, local_matrix_vector, locale_idx_of)  # noqa: F401
from .eigensolver import lobpcg  # noqa: F401
from .distributed import (DistributedOperator, EmulatedCluster, HostExchangedProduct,  # noqa: F401
                          HostReplicatedProduct, block_to_hashed, hashed_to_block, masks_of,
                          matrix_vector_product)

__all__ = [
    "BasisSpec", "OperatorSpec", "load_config_from_yaml", "Operator", "Basis", "BatchedOperator", "ChapelKernels",
    "local_matrix_vector", "matrix_vector_product", "locale_idx_of", "DistributedOperator",
    "EmulatedCluster", "HostExchangedProduct", "HostReplicatedProduct", "block_to_hashed", "hashed_to_block",
    "masks_of", "lobpcg",
]
