// acl_b200/csrc/context.h -- host-side objects behind the opaque handles of include/aclb200.h.
#pragma once

#include <cuda_runtime.h>

#include <stdint.h>
#include <initializer_list>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/aclb200.h"
#include "base_pose_cache.h"
#include "layout.h"

struct aclb200_context
{
	int device = 0;
	int num_sms = 0;
	int max_dynamic_smem = 0;
	std::string last_error;
	uint64_t launch_count = 0;

	// scratch of the host-buffer convenience call
	void* d_scratch_requests = nullptr;
	size_t scratch_requests_bytes = 0;
	void* d_scratch_out = nullptr;
	size_t scratch_out_bytes = 0;
	cudaStream_t host_stream = nullptr;
	cudaStream_t copy_stream = nullptr;			// device -> host copies of the host-buffer call overlap the next chunk's decode
	cudaEvent_t chunk_done[2] = { nullptr, nullptr };

	// aclb200_calculate_compression_error (error_metric.cu): job table, arg max accumulators, requests and the decoded poses of one chunk
	void* d_error_scratch = nullptr;
	size_t error_scratch_bytes = 0;
	cudaEvent_t error_scratch_done = nullptr;	// recorded after the last kernel of a call that reads the scratch, on that call's stream
	uint64_t error_chunk_bytes = 1024ull << 20;	// decoded poses per chunk (aclb200_set_error_chunk_bytes)

	// aclb200_debug_set_trace
	unsigned long long* d_trace = nullptr;
	uint32_t trace_blocks = 0;
	uint32_t trace_iterations = 0;

	// aclb200_debug_last_launch: the plan of the latest aclb200_decompress_tracks
	aclb200_launch_info last_launch = {};
};

namespace aclb200
{
	// One cached base pose variant of a clip set (pipeline.cu); its key and pins are kept by BasePoseCache (base_pose_cache.h)
	struct BasePoseRows
	{
		uint8_t* d_rows = nullptr;			// [num_clips][row_stride]
		uint32_t row_stride = 0;
		cudaEvent_t ready = nullptr;		// recorded after the build kernel on the stream that asked for it first
		cudaEvent_t last_launch = nullptr;	// recorded after the latest launch that reads the rows, on that launch's stream
	};
}

struct aclb200_clipset
{
	int device = 0;
	aclb200_clipset_info info = {};
	std::vector<aclb200::ClipDesc> host_clips;		// host mirror for the info queries
	std::vector<uint32_t> host_looping;				// compressed_tracks::get_looping_policy() per clip
	uint32_t max_animated[3] = { 0, 0, 0 };			// largest number of animated rotation / translation / scale sub-tracks of a clip
	uint32_t max_animated_total = 0;
	uint32_t max_key_frame_bytes = 0;				// largest ceil(animated_pose_bit_size / 8) of any segment
	bool all_tracks_even = true;					// every clip has an even number of tracks (40 byte bones then give 16 byte granular rows)

	uint8_t* d_data = nullptr;
	aclb200::ClipDesc* d_clips = nullptr;

	// aclb200_clipset_bind_database (database.cpp)
	const aclb200_database* database = nullptr;
	uint32_t* d_db_first_segment = nullptr;			// [num_clips] first database segment of each clip, 0xFFFFFFFF when it has none
	std::vector<uint32_t> host_blob_db_offset;		// [num_clips] clip_header_offset of its tracks_database_header, 0xFFFFFFFF without one
	std::vector<std::vector<uint32_t>> host_db_pose_bits;	// animated_pose_bit_size of each segment of the clips bound to a database

	// base pose rows built on first use per (layout, normalisation, default modes, constant default values), a handful kept, under
	// base_mutex
	mutable std::mutex base_mutex;
	mutable aclb200::BasePoseCache<aclb200::BasePoseRows> base_poses;
};

// A compressed_database on the device (database.cpp): the blob's headers stay on the host, the tier metadata and the streamed in
// bulk data live in HBM.
struct aclb200_database
{
	int device = 0;
	std::vector<uint8_t> blob;						// the compressed_database buffer (with its inline bulk data, if any)
	aclb200_database_info info = {};
	std::vector<uint32_t> clip_hash;				// per database clip, in runtime header order
	std::vector<uint32_t> clip_header_offset;		// runtime clip header offset of each clip (database_clip_metadata::clip_header_offset)
	std::vector<uint32_t> clip_first_segment;		// first database segment of each clip
	std::vector<uint32_t> clip_num_segments;
	mutable std::vector<uint32_t> segment_pose_bits;	// animated_pose_bit_size of each database segment once a clip set bound it, else 0
	std::vector<uint64_t> host_tiers;				// [num_segments][2] host mirror of d_tiers
	std::vector<uint32_t> loaded[2];				// loaded chunk bit sets, bit (31 - i % 32) of word i / 32 (acl::bitset)
	std::vector<std::vector<uint32_t>> chunk_segments[2];	// per tier and chunk: the segments whose metadata the streamed in chunk published
	unsigned long long* d_tiers = nullptr;			// [num_segments][2] database_runtime_segment_header::tier_metadata
	uint8_t* d_bulk[2] = { nullptr, nullptr };		// tier buffers (allocated while a chunk of the tier is streamed in)
};

namespace aclb200
{
	aclb200_status set_error(aclb200_context* context, aclb200_status status, const std::string& message);
	aclb200_status check_cuda(aclb200_context* context, cudaError_t error, const char* what);
	// api.cpp: zeroes *d_out_flags (when given) on the stream, before a launch that ORs ACLB200_ERROR_FLAG_* into it
	aclb200_status clear_out_flags(aclb200_context* context, uint32_t* d_out_flags, cudaStream_t stream, const char* what);
	// api.cpp: the pose buffers of a pose operation are rtm::qvvf rows: `pose_stride` (0 on entry: packed rows, set to num_tracks * 48)
	// holds num_tracks 48 byte bones and keeps them, like every pointer, 16 byte aligned
	aclb200_status check_qvvf_rows(aclb200_context* context, std::initializer_list<const void*> poses, uint32_t num_tracks, uint64_t& pose_stride,
		const char* what);
	// api.cpp: inverse bind matrices are 12 floats per skeleton entry, 16 byte aligned (each lane loads its bone's as three float4)
	aclb200_status check_inverse_binds(aclb200_context* context, const float* d_inverse_bind, const char* what);
	// database.cpp: the clip set is bound to a database with at least one chunk streamed in (the launch takes the database kernels)
	bool database_streamed_in(const aclb200_clipset* clipset);

	// One launch description shared by every kernel of the transform / scalar paths.
	struct DecodeParams
	{
		const uint8_t* data;
		const ClipDesc* clips;
		const aclb200_request* requests;
		const uint32_t* track_indices;		// decompress_track only
		uint32_t num_requests;
		uint32_t num_clips;
		uint32_t max_tracks;
		uint32_t max_animated[3];
		uint32_t requests_per_block;		// whole requests handled by one thread block
		uint32_t magic_tracks;				// floor(2^32 / d) + 1 for d = max_tracks / max_animated[0] / max(max_animated[1] + [2]):
		uint32_t magic_rot;					// turns slot / d into a mulhi (0 when d == 1)
		uint32_t magic_vec;
		uint32_t magic_chunks;
		uint32_t stage_bytes;				// shared memory bytes reserved per staged key frame (0 = read the streams from global memory)
		uint32_t smem_pose_bytes;			// shared memory bytes reserved per assembled pose (0 = phases store straight to global memory)
		uint32_t smem_stage_offset;			// carve-up of the dynamic shared memory: ReqState[] | key frame windows | poses
		uint32_t smem_out_offset;
		uint32_t smem_bytes;				// dynamic shared memory of the launch
		uint32_t out_vector16;				// poses can leave shared memory with 16 byte stores
		uint32_t out_bulk;					// pipeline: every pose row is 16 byte granular, rows leave shared memory as TMA bulk stores
		uint32_t grid_blocks;				// pipeline: persistent grid size
		uint32_t smem_stage_size;			// pipeline: bytes of one stage (key frame windows + poses)
		uint32_t hot_slot_bytes;			// pipeline: bytes of one slot of the ReqHot ring (records + group words)
		uint32_t smem_tag_offset;			// pipeline: base row tags (which clip's base pose each pose row holds)
		unsigned long long* trace;			// pipeline, ACLB200_PIPE_TRACE builds: clock stamps per (block, iteration), see aclb200_debug_set_trace
		uint32_t trace_blocks;
		uint32_t trace_iterations;
		const uint8_t* base_poses;			// pipeline: base pose row per clip (nullptr: phase A runs in the kernel)
		uint32_t base_stride;
		uint8_t* out;
		uint64_t pose_stride;
		uint32_t bone_stride;				// 48 or 40 (transform), components * 4 (scalar)

		uint32_t rounding_policy;
		uint32_t looping_policy;
		uint32_t normalization;
		uint32_t per_track_rounding;
		uint32_t wrapping;
		uint32_t clamp_sample_time;
		uint32_t multiple_rotation_formats;
		uint32_t default_mode[3];
		float    constant_defaults[12];
		const float* variable_defaults;
		const uint8_t* per_track_policies;
		uint32_t skip_all;					// ACLB200_SKIP_* bits skipped for every track
		const uint8_t* skip_tracks;			// [max_tracks] ACLB200_SKIP_* bits per track, or nullptr
		const uint8_t* request_policies;	// [num_requests][2] { rounding, looping } per request, or nullptr
		uint32_t layout;
		uint32_t debug_which;
		uint32_t debug_max_sub_tracks;
		// the database kernels (a clip set bound to a database with chunks streamed in, database.cpp)
		const uint32_t* db_first_segment;			// [num_clips] the clip's first database segment, 0xFFFFFFFF when it has none
		const unsigned long long* db_tiers;			// [database segments][2] tier metadata: (samples_offset << 32) | sample_indices
		const uint8_t* db_bulk[2];					// medium, low tier buffers
		// the object space decode (aclb200_decompress_tracks_object_space)
		const uint32_t* parent_indices;				// skeletons, 0xFFFFFFFF = root
		const uint32_t* skeleton_offsets;			// [num_clips] first parent index of each clip's skeleton, or nullptr (every clip at 0)
		uint32_t* object_flags;						// ACLB200_ERROR_FLAG_* are OR-ed in, or nullptr
		uint32_t object_kind;						// ACLB200_OBJECT_*, or k_object_skinning (the skinning decodes)
		const float* inverse_bind;					// k_object_skinning: one 12 float matrix per skeleton entry, in parallel with parent_indices
		// the additive decode (aclb200_decompress_tracks_additive): requests 2r / 2r + 1 are the base / additive halves of pair r, output r;
		// parent_indices == nullptr there keeps the combined poses in local space
		const uint8_t* clip_additive_formats;		// [num_clips] acl::additive_clip_format8 per additive clip (above 3: none), or nullptr
		uint32_t additive_format;					// the format when clip_additive_formats == nullptr
		// the blend decode (aclb200_decompress_tracks_blend): requests 2r / 2r + 1 are the from / to halves of pair r, output r
		const float* blend_weights;					// [pairs] the weight of each pair, or nullptr
		float blend_weight;							// the weight when blend_weights == nullptr
		// the layered decode (aclb200_decompress_tracks_layered): `requests` holds aclb200_layer records, requests r L .. r L + L - 1 are
		// the layers of output r (additive_format and clip_additive_formats as above)
		uint32_t num_layers;						// L, 1..k_max_layers
		uint32_t magic_layers;						// division_magic(L), for block-local indices
		// the masked layered decode (aclb200_decompress_tracks_layered_masked, k_compose_layers_masked)
		const uint32_t* layer_masks;				// [num_requests] the mask index of each layer (ACLB200_LAYER_NO_MASK: none), or nullptr
		const float* bone_masks;					// [num_masks][mask_stride] one weight per bone of the base clip
		uint32_t num_masks;							// at most k_max_layer_masks
		uint32_t mask_stride;
		// the inertialized decode (aclb200_decompress_tracks_inertialized, k_compose_inertialize): `requests` holds 20 byte
		// aclb200_inertialized_request records
		const uint8_t* records;						// record r at records + r * record_stride, 64 bytes per bone
		uint64_t record_stride;
		uint32_t num_records;						// < 2^32 - 1
		// the mirrored decode (aclb200_decompress_tracks_mirrored, k_compose_mirror): `requests` holds 12 byte aclb200_mirrored_request
		// records; clip c's table at mirror_table + skeleton_offsets[c]
		const aclb200_mirror_entry* mirror_table;
		uint32_t mirror_axis;						// ACLB200_MIRROR_*
	};

	// The bone query (aclb200_decompress_bones, bones.cu): the lists, the skeletons and the launch's shared memory carve-up. A kernel
	// argument of its own beside DecodeParams, which the other kernels share unchanged.
	struct BoneQuery
	{
		const uint32_t* bone_lists;				// [num_lists][bones_per_list] bone indices, ACLB200_NO_BONE for a hole
		const uint32_t* request_lists;			// [num_requests] the list of each request, or nullptr (every request takes list 0)
		uint32_t num_lists;
		uint32_t bones_per_list;				// K, 1..ACLB200_MAX_QUERY_BONES
		const uint32_t* parent_indices;			// skeletons (object space rows), or nullptr (local rows)
		const uint32_t* skeleton_offsets;		// [num_clips] first parent index of each clip's skeleton, or nullptr
		uint32_t object_kind;					// ACLB200_OBJECT_QVVF or ACLB200_OBJECT_MATRIX3X4F, with parents
		uint32_t* out_flags;					// ACLB200_ERROR_FLAG_* of the walked bones are OR-ed in, or nullptr
		uint32_t requests_per_block;
		uint32_t mask_words;					// closure bitmask words per request: ceil(max_tracks / 32)
		uint32_t smem_pose_bytes;				// pose rows per request: max_tracks * bone size, 16 byte granular
		uint32_t smem_words_offset;				// dynamic shared memory: request states | request words | closure bitmasks | work items |
		uint32_t smem_mask_offset;				// pose rows
		uint32_t smem_items_offset;
		uint32_t smem_pose_offset;
		uint32_t smem_bytes;
	};

	// Root motion (aclb200_extract_root_motion, root_motion.cu): the requests and the root track of each clip. A kernel argument of its own
	// beside DecodeParams, whose `requests` it leaves unused (each lane builds its own request from the root motion request's times).
	struct RootMotionQuery
	{
		const aclb200_root_motion_request* requests;
		const uint32_t* root_tracks;			// [num_clips] the root track of each clip, or nullptr (track 0)
		uint32_t* out_flags;					// ACLB200_ERROR_FLAG_NEGATIVE_SCALE and ACLB200_ERROR_FLAG_WRAP_CLIP_CYCLE are OR-ed in, or nullptr
	};

	// The pose features (aclb200_extract_pose_features, features.cu): a third kernel argument beside DecodeParams and the bone query's
	// BoneQuery. The launch runs the bone query's plan on virtual requests r * num_offsets + s (request r at offset s): DecodeParams'
	// num_requests counts them and its `requests` is unused.
	struct FeatureQuery
	{
		const aclb200_feature_request* requests;
		const uint32_t* root_tracks;			// [num_clips] the root track of each clip, or nullptr (track 0)
		float offsets[ACLB200_MAX_FEATURE_OFFSETS];
		uint32_t num_offsets;					// S, 1..ACLB200_MAX_FEATURE_OFFSETS
	};

	// The pack (aclb200_pack_pose_features, feature_search.cu): each output dimension resolved from its term on the host
	struct PackDim
	{
		uint32_t kind;							// ACLB200_FEATURE_POSITION / DIRECTION / VELOCITY
		uint32_t row0;							// s0 * K + k: the row read (VELOCITY: subtracted)
		uint32_t row1;							// VELOCITY: s1 * K + k
		uint32_t component;						// 0, 1, 2 = x, y, z
		uint32_t axis;							// DIRECTION: the unit axis rotated
		float inv_dt;							// VELOCITY
		float mean;
		float scale;
	};
	struct PackParams
	{
		const uint8_t* rows;					// request r's rows at rows + r * pose_stride, 48 bytes each
		uint64_t pose_stride;
		float* out;								// request r's vector at out + r * out_stride
		uint64_t out_stride;					// floats
		uint32_t num_requests;
		uint32_t num_dims;
		PackDim dims[ACLB200_MAX_FEATURE_DIMS];
	};

	// The search (aclb200_search_pose_features, feature_search.cu)
	struct SearchParams
	{
		const float* database;					// row r at database + r * db_stride
		const float* query_vectors;				// query q at query_vectors + q * q_stride
		const aclb200_search_query* queries;
		const uint32_t* row_tags;				// [num_rows], or nullptr (every tag 0xFFFFFFFF)
		aclb200_search_result* results;
		uint64_t num_rows;						// N < 2^32 - 1
		uint64_t db_stride;						// floats
		uint64_t q_stride;
		uint32_t num_queries;
		uint32_t num_dims;
	};

	// The inertialization capture (aclb200_begin_inertialization, inertialization.cu): transition j's four QVV48 poses at j * pose_stride,
	// its record at records + (record_slots ? record_slots[j] : j) * record_stride, 64 bytes per bone
	struct InertializationCapture
	{
		const uint8_t* src;
		const uint8_t* src_prev;
		const uint8_t* dst;
		const uint8_t* dst_prev;
		uint8_t* records;
		const uint32_t* record_slots;
		uint64_t num_transitions;
		uint64_t pose_stride;
		uint64_t record_stride;
		uint32_t num_tracks;
		float inv_dt;
	};

	// The inertialization apply (aclb200_inertialize_poses, inertialization.cu): pose p at p * pose_stride in poses and out, decayed with
	// inertializations[p]
	struct InertializationApply
	{
		const uint8_t* poses;
		uint8_t* out;
		const aclb200_inertialization* inertializations;
		const uint8_t* records;
		uint64_t num_poses;
		uint64_t pose_stride;
		uint64_t record_stride;
		uint64_t num_records;					// < 2^32 - 1
		uint32_t num_tracks;
	};

	// The pose mirror (aclb200_mirror_poses, mirror.cu): pose p at p * pose_stride in poses and out, row i mirrored with table[i]
	struct MirrorApply
	{
		const uint8_t* poses;
		uint8_t* out;
		const uint32_t* mirrored;				// [num_poses] 0 copy, 1 mirror, other: not written; NULL: every pose mirrored
		const aclb200_mirror_entry* table;
		uint32_t* flags;
		uint64_t num_poses;
		uint64_t pose_stride;
		uint32_t num_rows;
		uint32_t axis;
	};

	// What transform_decompress_tracks_kernel makes of its poses before they leave. local: the decoded poses (aclb200_decompress_tracks).
	// object: taken to object space (aclb200_decompress_tracks_object_space). additive, blend: pair r is requests 2r and 2r + 1, combined
	// into output r (aclb200_decompress_tracks_additive / _blend). layers: stack r is requests r L .. r L + L - 1, folded into output r
	// (aclb200_decompress_tracks_layered). layers_masked: the layers mode with bone masks and weighted ADDITIVE layers
	// (aclb200_decompress_tracks_layered_masked). inertialize: each request's pose with its inertialization record's offset decayed onto
	// it (aclb200_decompress_tracks_inertialized). mirror: each request's pose, mirrored when its request asks (aclb200_decompress_tracks_mirrored).
	enum : uint32_t { k_compose_local = 0, k_compose_object = 1, k_compose_additive = 2, k_compose_blend = 3, k_compose_layers = 4,
		k_compose_layers_masked = 5, k_compose_inertialize = 6, k_compose_mirror = 7, k_compose_count = 8 };

	// the deepest layer stack of aclb200_decompress_tracks_layered
	constexpr uint32_t k_max_layers = 8;

	// the most bone masks of one aclb200_decompress_tracks_layered_masked launch: a layer's slot keeps its mask index + 1 in the 29 bits
	// above its op
	constexpr uint32_t k_layer_op_bits = 3;
	constexpr uint32_t k_max_layer_masks = (1u << (32 - k_layer_op_bits)) - 1;

	// The object kind of the skinning decodes (after ACLB200_OBJECT_QVVF and ACLB200_OBJECT_MATRIX3X4F, never taken from a caller): the
	// matrix walk, then rtm::matrix_mul(inverse_bind, object) per bone, stored as the transposed rows a skinning shader reads
	constexpr uint32_t k_object_skinning = 2;

	// kernels.cu
	// every mode but local assembles its poses in shared memory; additive and blend plan whole pairs, layers whole stacks of
	// params.num_layers requests
	void plan_launch(DecodeParams& params, uint32_t max_key_frame_bytes, int max_dynamic_smem, bool allow_output_staging, bool database,
		uint32_t compose);
	void plan_scalar_launch(DecodeParams& params, uint32_t max_key_frame_bytes);
	cudaError_t launch_transform_decompress_tracks(const DecodeParams& params, uint32_t compose, bool database, cudaStream_t stream);
	cudaError_t launch_transform_decompress_track(const DecodeParams& params, bool database, cudaStream_t stream);
	cudaError_t launch_apply_additive(const uint8_t* base_poses, const uint8_t* additive_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
		uint64_t pose_stride, uint32_t additive_format, uint32_t* flags, int num_sms, cudaStream_t stream);
	cudaError_t launch_blend_poses(const uint8_t* from_poses, const uint8_t* to_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
		uint64_t pose_stride, float weight, const float* weights, int num_sms, cudaStream_t stream);
	// the grid of the pose operations: one thread per (pose, bone), at most 16 blocks of 256 threads per SM, which loop over the rest
	uint32_t pose_operation_blocks(uint64_t num_poses, uint32_t num_tracks, int num_sms);
	// aclb200_local_to_skinning: one warp per pose, the pose staged in shared memory; 0 warps per block when one pose does not fit
	uint32_t local_to_skinning_warps(uint32_t num_tracks, int max_dynamic_smem);
	cudaError_t launch_local_to_skinning(const uint8_t* local_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride,
		const uint32_t* parents, const float* inverse_bind, uint32_t* flags, uint32_t warps, int num_sms, cudaStream_t stream);
	cudaError_t launch_transform_debug_seek(const DecodeParams& params, aclb200_seek_state* d_out, cudaStream_t stream);
	cudaError_t launch_transform_debug_unpack(const DecodeParams& params, uint32_t* d_out, cudaStream_t stream);
	cudaError_t launch_scalar_decompress_tracks(const DecodeParams& params, cudaStream_t stream);
	cudaError_t launch_scalar_decompress_track(const DecodeParams& params, cudaStream_t stream);
	cudaError_t configure_kernels(int& max_dynamic_smem);
	// bones.cu: the bone query. plan_bones_launch returns false when one request does not fit max_dynamic_smem; `extra_request_bytes`
	// (16 byte granular) per request follow the pose rows (the pose features' root samples).
	cudaError_t configure_bones_kernels(int max_dynamic_smem);
	bool plan_bones_launch(const DecodeParams& params, BoneQuery& query, bool database, int max_dynamic_smem, uint32_t extra_request_bytes = 0);
	cudaError_t launch_decompress_bones(const DecodeParams& params, const BoneQuery& query, bool database, cudaStream_t stream);
	// root_motion.cu: root motion, one lane per (request, sample)
	cudaError_t launch_extract_root_motion(const DecodeParams& params, const RootMotionQuery& query, bool database, cudaStream_t stream);
	// features.cu: the pose features, on the bone query's plan (plan_features_launch: false when one pose does not fit max_dynamic_smem)
	cudaError_t configure_features_kernels(int max_dynamic_smem);
	bool plan_features_launch(const DecodeParams& params, BoneQuery& query, bool database, int max_dynamic_smem);
	cudaError_t launch_extract_pose_features(const DecodeParams& params, const BoneQuery& query, const FeatureQuery& features, bool database,
		cudaStream_t stream);
	// feature_search.cu: the pack, one thread per output float; the search, which writes every result then atomicMin-s each block's best
	cudaError_t configure_feature_search_kernels();
	cudaError_t launch_pack_pose_features(const PackParams& params, cudaStream_t stream);
	cudaError_t launch_search_pose_features(const SearchParams& params, int num_sms, cudaStream_t stream);
	// inertialization.cu: the capture and the apply, one thread per (pose, bone)
	cudaError_t launch_begin_inertialization(const InertializationCapture& capture, int num_sms, cudaStream_t stream);
	cudaError_t launch_inertialize_poses(const InertializationApply& apply, int num_sms, cudaStream_t stream);
	// mirror.cu: one thread per (pose, partner pair)
	cudaError_t launch_mirror_poses(const MirrorApply& apply, int num_sms, cudaStream_t stream);
	// error_metric.cu
	cudaError_t configure_error_kernels(int optin_limit);
	// pipeline.cu
	cudaError_t configure_pipeline_kernels(int optin_limit, int& min_available);
	bool plan_pipeline(DecodeParams& params, uint32_t max_key_frame_bytes, int max_dynamic_smem, int num_sms);
	cudaError_t launch_transform_pipeline(const DecodeParams& params, uint32_t math_mode, cudaStream_t stream);
	void acquire_base_poses(const aclb200_clipset* clipset, DecodeParams& params, cudaStream_t stream);
	void release_base_poses_use(const aclb200_clipset* clipset, const DecodeParams& params, cudaStream_t stream);
	void release_base_poses(aclb200_clipset* clipset);
}
