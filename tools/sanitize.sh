# compute-sanitizer over small invocations of every kernel family (memcheck everywhere, racecheck on the shared-memory heavy ones)
set -x
export SHINE_UNDER_SANITIZER=1
SEL="grouped_scatter or capture_step or ragged_batch_sizes and 17 or fused_step_matches_oracle and 2-True or adam_kernel or fused_eikonal_step_matches_oracle and 2-True or regularization_and_importance or three_ranges or cuda_update_matches or hash_insert_reports or add_frame_equals_oracle and 2049 or several_frames_compact or pool_window_append_rejects or append_across_chunk_boundaries or get_batch_equals_sample_pool and 4096 or first_and_last_record_of_every_chunk or pool_past_four_gigabytes or get_batch_in_a_cuda_graph or host_pool_rejects_bad_input"
timeout 1500 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests -m gpu -q -k "$SEL" 2>&1 | tail -8
timeout 1200 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -m gpu -q -x -k "fused_step_matches_oracle and 2-True or fused_eikonal_step_matches_oracle and 2-True or grouped_scatter_matches_oracle and 3-True-False-mean-True or grouped_scatter_dense" 2>&1 | tail -6
timeout 1200 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_replay.py -m gpu -q -x -k "add_frame_equals_oracle and 2049 or several_frames_compact" 2>&1 | tail -6
