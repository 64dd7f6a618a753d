#!/bin/bash
# compute-sanitizer passes (run on a GPU box; minutes): the class pipeline, the cooperative kernel (TMA + mbarrier, at 16-
# and 64-token blocks), the two-phase write path with its slot-ownership protocol.
set -x
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "prefix_tree and classes8"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "alphabet and classes8 and 1"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_concurrency.py -x -q -m gpu -k "coop_kernel_short or two_phase or duplicate_hashes"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_concurrency.py -x -q -m gpu -k "coop_kernel_short"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "ragged and coop"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "test_random_event_stream and rounds"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "prefix_tree and rounds2 and not lane"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_snapshot.py -x -q -m gpu -k "golden or error_paths or equal_contents or exact_lru"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_shard_ops.py -x -q -m gpu -k "same-gpu-2 or guards or all_or_nothing or unsharded_handle or (round_trips and coop and same)"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_score_keys.py -x -q -m gpu -k "same_bits or arbitrary or host_buffers or errors"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_score_keys.py -x -q -m gpu -k "arbitrary and 257"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_score_turn.py -x -q -m gpu -k "identities or arbitrary or chain_edges or block_sizes or host_buffers or errors"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_score_turn.py -x -q -m gpu -k "chain_edges or (arbitrary and 257)"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_host_buffers.py -x -q -m gpu -k "model_filter or exact_lru"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_inventory.py -x -q -m gpu -k "max_pods or removing_each_pod or high_load or shard_inventories or errors"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_inventory.py -x -q -m gpu -k "max_pods and (257 or 513)"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_block_sizes.py -x -q -m gpu -k "payloads_and_shapes and 64-None"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_block_sizes.py -x -q -m gpu -k "payloads_and_shapes and 64-None"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_lru_recency.py -x -q -m gpu -k "lookup or add or events or (shared_prefixes and 16 and (dense or dev or keys or turn))"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_text_store.py -x -q -m gpu -k "hash_chains or (call_streams and (7 or 1000)) or arena or enospc or slices or errors or (score_text and default and (-1] or -32] or -2048]))"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_text_store.py -x -q -m gpu -k "hash_chains and 37"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_text_store_scale.py -x -q -m gpu -k "grows_the_arena or (index_block_sizes and 32-2048) or queued_behind or clock_bits"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_pinned_staging.py -x -q -m gpu
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_lookup_hits.py -x -q -m gpu -k "(against_the_oracle and (257 or 4096)) or long_prompt or (tokens_form and 4) or (at_scale and (1] or 33])) or errors"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_lookup_hits.py -x -q -m gpu -k "(against_the_oracle and 257 and random) or (long_prompt and False)"
