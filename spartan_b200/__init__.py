"""spartan_b200 — H100-native prover for the Spartan zkSNARK (drop-in for the prover hot path of microsoft/Spartan).

The product is the C-ABI library `libspartan_b200.so` (include/spartan_b200.h): hand-written sm_90a kernels plus a C++ host
prover.  This package is a thin ctypes mirror of the reference's public API (src/lib.rs): Instance, Assignment, NIZKGens, NIZK,
SNARKGens, SNARK — same names, argument meaning and error behaviour.  There is no CPU fallback: without the CUDA library or
without a GPU every entry point raises.
"""
from .api import (  # noqa: F401
    Assignment, Composition, Context, DensePolynomial, GeneratorTables, InputsAssignment, Instance, MultiCommitGens, NIZK, NIZKGens, ProofVerifyError, R1CSError, SNARK,
    SNARKGens, SpartanB200Error, Transcript, VarsAssignment, default_context, device_bytes_live, kernel_launches, lib, random_tape_seed, release_cached_memory, scalar_from_bytes, scalar_to_bytes, tape_seed, prg_scalars,
    sumcheck_prove, sumcheck_verify, debug_memcheck, debug_memcheck_report, debug_memcheck_scan,
    PolyCommitmentGens, PolyCommitment, PolyEvalProof, RandomTape, poly_commit,
    ZKSumcheckInstanceProof, KnowledgeProof, EqualityProof, ProductProof, DotProductProof, DotProductProofGens, DotProductProofLog,
    ProductLeaves, ProductCircuits, ProductCircuitEvalProofBatched, product_leaf_eval,
    SparseMatPolyCommitmentGens, SparseMatPolyCommitment, SparseMatPolyDense, SparseMatPolynomial, SparseMatPolyEvalProof,
    SparseMatProducts, R1CSGens, R1CSProof,
)
