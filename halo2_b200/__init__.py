"""halo2_b200 -- H100-native MSM + NTT engine behind halo2's best_multiexp / best_fft /
Params::commit* / EvaluationDomain transforms.

The compute path is the sm_90a CUDA library `_lib/libhalo2_b200.so` (C ABI:
include/halo2_b200.h).  There is no CPU fallback: importing works anywhere, but every
operation raises `H2Error` unless the library is built and an H100 is visible.
"""
from .lib import H2Error, Lane, lib_path, load, init, launch_count  # noqa: F401
from .arithmetic import (best_multiexp, small_multiexp, best_fft, best_fft_curve, batch_normalize, multiexp_window_bits,  # noqa: F401
                         eval_polynomial, compute_inner_product, kate_division)
from .poly import (Params, EvaluationDomain, Blind, ResidentPoly, lagrange_generators, compress_points, decompress_points, hash_to_curve,  # noqa: F401
                   eval_polynomial_resident, inner_product_resident, kate_division_resident, batch_invert_resident,
                   running_product_resident, permute_expression_pair_resident, share_resident, set_rows_resident,
                   upload_tensors_resident, download_tensors_resident, upload_dev_resident, download_dev_resident)

from .evaluator import Ast, AstLeaf, Evaluator  # noqa: F401
from .verifier import MSM, Guard, VerifyError, verify_proof, compute_b  # noqa: F401
from .keygen import (Assembly, CopyConstraints, ProvingKey, build_permutation_polys, keygen_vk, keygen_pk,  # noqa: F401
                     batch_invert_assigned_resident)
from .products import (permutation_commit, lookup_commit_product, permutation_product_resident, lookup_product_resident,  # noqa: F401
                       lookup_commit_permuted, lookup_permute_resident, Permuted)
from .columns import instance_commit, advice_commit, InstanceSingle, AdviceSingle, InstanceTooLarge  # noqa: F401
from .vanishing import vanishing_commit, vanishing_quotient_resident, Committed, Constructed, Evaluated  # noqa: F401
from .arguments import (PermutationCommitted, PermutationConstructed, PermutationEvaluated, permutation_key_evaluate,  # noqa: F401
                        permutation_key_open, LookupCommitted, LookupConstructed, LookupEvaluated, evaluate_columns, open_columns)
from .rng import ChaCha20Rng, random_resident  # noqa: F401
from . import multiopen, opening  # noqa: F401

__all__ = ["Ast", "AstLeaf", "Evaluator", "Assembly", "CopyConstraints", "ProvingKey", "build_permutation_polys", "keygen_vk", "keygen_pk",
           "batch_invert_assigned_resident", "MSM", "Guard", "VerifyError", "verify_proof", "compute_b", "multiopen", "opening", "H2Error", "Lane", "lib_path", "load", "init", "launch_count", "best_multiexp", "small_multiexp", "best_fft",
           "best_fft_curve", "batch_normalize", "multiexp_window_bits", "Params", "EvaluationDomain", "Blind", "ResidentPoly",
           "lagrange_generators", "compress_points", "decompress_points", "hash_to_curve",
           "eval_polynomial", "compute_inner_product", "kate_division", "eval_polynomial_resident", "inner_product_resident",
           "kate_division_resident", "batch_invert_resident", "running_product_resident", "permute_expression_pair_resident",
           "share_resident", "upload_tensors_resident", "download_tensors_resident", "upload_dev_resident", "download_dev_resident",
           "permutation_commit", "lookup_commit_product", "permutation_product_resident", "lookup_product_resident",
           "lookup_commit_permuted", "lookup_permute_resident", "Permuted", "set_rows_resident", "instance_commit", "advice_commit",
           "InstanceSingle", "AdviceSingle", "InstanceTooLarge",
           "vanishing_commit", "vanishing_quotient_resident", "Committed", "Constructed", "Evaluated",
           "PermutationCommitted", "PermutationConstructed", "PermutationEvaluated", "permutation_key_evaluate", "permutation_key_open",
           "LookupCommitted", "LookupConstructed", "LookupEvaluated", "evaluate_columns", "open_columns", "ChaCha20Rng", "random_resident"]
