"""plaid_b200: H100-native (sm_90a) PLAID search path behind next-plaid's MmapIndex interface.

The directory is named `next-plaid_b200` (the name the project brief fixes); import it as
`next_plaid_b200` through the shim module at the repository root.
"""
from .index import (MmapIndex, PlaidError, QueryResult, SearchParameters, SearchTrace, STAGES,
                    device_count, comm_unique_id, ShardGroup, load_library, ResidualCodec, kmeans_fit, create_index, create_index_sharded, last_create_ms, kmeans_sizing, kmeans_fit_dp, maxsim_scores, shard_bounds, LIB_PATH, EXPORTS,
                    pool_document_embeddings, pooled_doc_length, last_pool_ms)
from .build import build_library

__all__ = ["MmapIndex", "PlaidError", "QueryResult", "SearchParameters", "SearchTrace", "STAGES",
           "device_count", "comm_unique_id", "ShardGroup", "load_library", "ResidualCodec", "kmeans_fit", "create_index", "create_index_sharded", "last_create_ms", "kmeans_sizing", "kmeans_fit_dp", "maxsim_scores", "shard_bounds", "build_library", "LIB_PATH", "EXPORTS",
           "pool_document_embeddings", "pooled_doc_length", "last_pool_ms"]
