"""Engine tunables.  The names are the reference's (dampr/settings.py:5-37) so scripts that set
``settings.max_processes`` or ``settings.partitions`` keep working; the meanings are re-mapped to
the device engine (SURVEY §5 "Config / flags").
"""
import os

# reference: number of worker processes. here: host threads used for file ingest and host-side
# (non-lowered) map functions; the shuffle itself runs on the GPU(s).
max_processes = os.cpu_count() or 1

# reference: gzip level of spilled runs. here: unused (runs stay uncompressed in HBM / pinned host).
compress_level = 1

# reference: number of hash partitions (91). here: advisory; the device radix fan-out is chosen
# from the record count (csrc/kv.cu: sort_range).
partitions = 91

# reference: max run files per partition before a compaction pass. here: merge fan-in of spilled runs.
max_files_per_stage = 50

# reference: tuples per pickle frame. here: unused.
batch_size = 1000

memory_checker_type = "interpolative"

# reference: RSS growth (MB) that triggers a spill in a worker. here: device arena (MB) a single
# stage may hold before sorted runs are spilled to pinned host memory.
max_memory_per_worker = 512

memory_check_base = 1.2
memory_min_count = 10000
memory_max_count_before_check = 100000

# ---- additions of the device engine -------------------------------------------------------
# GPU used by a single-process run (multi-GPU runs take LOCAL_RANK)
device = int(os.environ.get("LOCAL_RANK", "0"))
# bytes per host->device ingest chunk of text inputs
ingest_chunk_bytes = 64 << 20
# log2 of the combiner table capacity (entries) for text counting
text_table_log2 = 21  # grows (x4) and the scan re-runs when it overflows or fills beyond 50 %
# device arena in bytes available to one sort before it spills runs (None = no cap)
device_arena_bytes = None
# the host buffer that holds the spilled runs of one job is kept for the next job when it is at most this large
# (its pages are then already mapped: no page faults on the way out, nothing to unmap at the end);
# spill.release_host_arena() returns it to the OS
host_spill_cache_bytes = 96 << 30
# page-locked host memory a device context keeps for result downloads (the token table, the count dictionary), and
# the bound on the sink's kept formatting buffers; a result larger than this is downloaded into pageable memory
host_result_cache_bytes = 64 << 20
# build of the tokenise kernel the scans start with: CTAs per SM it is sized for (4, 3 or 2; lines with more
# distinct tokens than a build remembers are retried on the 2-CTA build, see plan.TextScan.run)
text_kernel_ctas = 4
# host maps (stages whose lambdas are not lowered) over text files of at least this many bytes run in
# forked worker processes (settings.max_processes of them), like the reference's process pool
host_map_parallel_bytes = 16 << 20
# host reduces (reducers that are not lowered) over at least this many grouped records are split over forked
# workers at group boundaries
host_reduce_parallel_records = 500000
