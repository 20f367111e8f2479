/* include/aclb200.h -- C ABI of libaclb200.so: batched, H100-native (sm_90a) decompression of
 * nfrechette/acl `compressed_tracks` blobs.
 *
 * ACL (reference @ 0f855f0) has no FFI layer of its own: its "operator API" for this path is the
 * header-only C++ class acl::decompression_context<settings> (includes/acl/decompression/decompress.h:76-201)
 * driven by a duck-typed acl::track_writer (includes/acl/core/track_writer.h:82-216). The entry points
 * below are what a binding of that path needs, one (clip, sample_time) request per pose, many requests
 * per call. Each one names the reference interface it replaces. include/acl_b200/decompress.h is the C++
 * header shim that keeps the reference's class/method names on top of these functions, and
 * INTEGRATION.md shows the binding a maintainer would add on the reference side.
 *
 * Conventions: POD only, no C++ types, no exceptions; every function returns an aclb200_status;
 * device pointers are plain `void*` / typed pointers into CUDA device memory of the context's device;
 * `stream` is a `cudaStream_t` passed as `void*` (NULL = the legacy default stream). Calls are
 * asynchronous on `stream` unless stated otherwise. There is NO CPU fallback: without a CUDA device
 * aclb200_create fails with ACLB200_ERR_NO_DEVICE.
 */
#ifndef ACLB200_H
#define ACLB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
	#define ACLB200_API __declspec(dllexport)
#else
	#define ACLB200_API __attribute__((visibility("default")))
#endif

#define ACLB200_VERSION_MAJOR 0
#define ACLB200_VERSION_MINOR 17

typedef enum aclb200_status
{
	ACLB200_OK = 0,
	ACLB200_ERR_INVALID_ARGUMENT = 1,
	ACLB200_ERR_INVALID_CLIP = 2,		/* what decompression_context::initialize() reports by returning false (decompress.impl.h:66-83) */
	ACLB200_ERR_UNSUPPORTED = 3,		/* valid ACL data this build refuses: mixed track types in one clip set, clip images past 4 GiB */
	ACLB200_ERR_NO_DEVICE = 4,
	ACLB200_ERR_CUDA = 5,
	ACLB200_ERR_OUT_OF_MEMORY = 6
} aclb200_status;

/* acl::sample_rounding_policy (core/sample_rounding_policy.h:47-107) */
enum { ACLB200_ROUND_NONE = 0, ACLB200_ROUND_FLOOR = 1, ACLB200_ROUND_CEIL = 2, ACLB200_ROUND_NEAREST = 3, ACLB200_ROUND_PER_TRACK = 4 };
/* acl::sample_looping_policy (core/sample_looping_policy.h:56-82) */
enum { ACLB200_LOOP_CLAMP = 0, ACLB200_LOOP_WRAP = 1, ACLB200_LOOP_AS_COMPRESSED = 2 };
/* acl::rotation_normalization_policy_t (decompression/decompression_settings.h:52-62) */
enum { ACLB200_NORMALIZE_NEVER = 0, ACLB200_NORMALIZE_LERP_ONLY = 1, ACLB200_NORMALIZE_ALWAYS = 2 };
/* acl::default_sub_track_mode (core/track_writer.h:49-74) */
enum { ACLB200_DEFAULT_SKIPPED = 0, ACLB200_DEFAULT_CONSTANT = 1, ACLB200_DEFAULT_VARIABLE = 2, ACLB200_DEFAULT_LEGACY = 3 };
/* acl::track_type8 (core/track_types.h:53-68) */
enum { ACLB200_TRACK_FLOAT1F = 0, ACLB200_TRACK_FLOAT2F = 1, ACLB200_TRACK_FLOAT3F = 2, ACLB200_TRACK_FLOAT4F = 3, ACLB200_TRACK_VECTOR4F = 4, ACLB200_TRACK_QVVF = 12 };

/* Output layouts of the transform path (the device-side stand-in for track_writer::write_rotation/translation/scale). */
enum
{
	ACLB200_LAYOUT_QVV48 = 0,	/* rtm::qvvf as debug_track_writer stores it: rotation xyzw, translation xyz + 0, scale xyz + 0 (48 B / bone) */
	ACLB200_LAYOUT_QVV40 = 1	/* rotation xyzw, translation xyz, scale xyz (40 B / bone) == the reference's own "pose size"
								 * (tools/acl_decompressor/sources/benchmark.cpp:146-147) */
};

/* Arithmetic of the float stage. The integer / format decode is bit-exact in both modes. */
enum
{
	ACLB200_MATH_EXACT = 0,		/* IEEE-754 mul/add/sqrt/div in the reference's operation order, never fused: bit-identical
								 * to the reference's SSE2/AVX/scalar builds for decompress_tracks */
	ACLB200_MATH_FAST = 1		/* decompress_tracks on variable bit rate rotations: x, y, z and the W reconstruction input stay exact,
								 * then hardware sqrt / rsqrt and fused multiply-adds: rotations <= 1e-5 absolute from EXACT
								 * (including W ~ 0), translations / scales / every other path unchanged (bit-exact) */
};

typedef struct aclb200_context aclb200_context;
typedef struct aclb200_clipset aclb200_clipset;
typedef struct aclb200_database aclb200_database;

/* One decompression request == one `context.initialize(clip); context.seek(sample_time, policy);
 * context.decompress_tracks(writer);` sequence of the reference (decompress.h:90-172). */
typedef struct aclb200_request
{
	uint32_t clip;				/* index into the clip set */
	float    sample_time;		/* seconds, clamped to the clip like seek() does (decompression.transform.h:215-216) */
} aclb200_request;

/* Everything the reference bakes into `decompression_settings` (decompression_settings.h:74-166) and
 * `track_writer` (track_writer.h:82-216) at compile time, plus the seek() arguments shared by the batch.
 * Zero-initialise then call aclb200_default_options(). */
typedef struct aclb200_options
{
	uint32_t struct_size;					/* sizeof(aclb200_options), for forward compatibility */

	/* seek(sample_time, rounding_policy) + set_looping_policy(policy) (decompress.h:147-160) */
	uint32_t rounding_policy;				/* ACLB200_ROUND_* */
	uint32_t looping_policy;				/* ACLB200_LOOP_* */

	/* decompression_settings */
	uint32_t normalization;					/* get_rotation_normalization_policy() */
	uint32_t per_track_rounding;			/* is_per_track_rounding_supported() */
	uint32_t wrapping;						/* is_wrapping_supported() */
	uint32_t clamp_sample_time;				/* clamp_sample_time() */
	uint32_t multiple_rotation_formats;		/* more than one is_rotation_format_supported(): only changes the result for quatf_full
											 * clips sampled exactly on a key frame (decompression_context.transform.h:191-200) */

	/* track_writer */
	uint32_t default_rotation_mode;			/* get_default_rotation_mode(): ACLB200_DEFAULT_* (legacy is scale only) */
	uint32_t default_translation_mode;
	uint32_t default_scale_mode;
	float    constant_defaults[12];			/* get_constant_default_rotation/translation/scale(): xyzw, xyz-, xyz- */
	const float* d_variable_defaults;		/* get_variable_default_*(track): device [max_tracks][12] floats, or NULL */
	const uint8_t* d_per_track_rounding;	/* get_rounding_policy(per_track, track): device [max_tracks] ACLB200_ROUND_*, or NULL */

	/* output */
	uint32_t output_layout;					/* ACLB200_LAYOUT_* */
	uint32_t math_mode;						/* ACLB200_MATH_* */
	uint64_t pose_stride_bytes;				/* distance between the poses of consecutive requests; 0 = max_tracks * bone size */

	/* track_writer::skip_all_rotations/translations/scales() and skip_track_rotation/translation/scale(track)
	 * (core/track_writer.h:181-191, honoured per sub-track at decompression.transform.h:626-665 and in every unpack pass):
	 * a skipped sub-track is NOT written, the output buffer keeps what it held. Transform clip sets only. */
	uint32_t skip_mask;						/* ACLB200_SKIP_* bits: sub-track kinds skipped for every track */
	const uint8_t* d_skip_track_mask;		/* device [max_tracks] bytes of ACLB200_SKIP_* bits: sub-tracks skipped per track, or NULL */

	/* seek(sample_time, rounding_policy) / set_looping_policy(policy) PER REQUEST (the reference takes both per call,
	 * decompress.h:147-160): device [num_requests][2] bytes { ACLB200_ROUND_* (none..nearest), ACLB200_LOOP_* }, or NULL to use
	 * rounding_policy / looping_policy above for the whole batch. Values out of range read as none / as_compressed;
	 * ACLB200_ROUND_PER_TRACK stays a batch wide choice (rounding_policy + d_per_track_rounding). */
	const uint8_t* d_request_policies;
} aclb200_options;

enum { ACLB200_SKIP_ROTATION = 1, ACLB200_SKIP_TRANSLATION = 2, ACLB200_SKIP_SCALE = 4 };

typedef struct aclb200_clipset_info
{
	uint32_t num_clips;
	uint32_t track_type;			/* ACLB200_TRACK_*: a clip set holds transform clips or scalar clips of one type, never both */
	uint32_t max_tracks;
	uint32_t min_tracks;
	uint64_t blob_bytes;			/* device bytes holding the compressed clips */
	uint64_t index_bytes;			/* device bytes of the acceleration index built at upload */
} aclb200_clipset_info;

typedef struct aclb200_clip_info
{
	uint32_t num_tracks;
	uint32_t num_samples;
	float    sample_rate;
	float    duration;				/* compressed_tracks::get_finite_duration() with the clip's own looping policy */
	uint32_t num_segments;
	uint32_t looping_policy;		/* compressed_tracks::get_looping_policy() */
	uint32_t hash;					/* compressed_tracks::get_hash() */
	uint32_t size;
} aclb200_clip_info;

/* Device-side result of seek(), exposed for integer parity checks against the reference
 * (persistent_transform_decompression_context_v0, decompression_context.transform.h:53-116). */
typedef struct aclb200_seek_state
{
	float    sample_time;			/* clamped; < 0 when the request was invalid */
	float    interpolation_alpha;
	uint32_t key_frame_bit_offsets[2];
	uint32_t segment_indices[2];
	uint32_t animated_offsets[2];	/* byte offsets of the animated bit streams relative to the start of the clip */
	uint32_t format_offsets[2];
	uint32_t range_offsets[2];
	uint32_t uses_single_segment;
	uint32_t looping_policy;
} aclb200_seek_state;

ACLB200_API const char* aclb200_version_string(void);
ACLB200_API const char* aclb200_status_string(aclb200_status status);

/* Fills `options` with default_transform_decompression_settings + acl::track_writer defaults
 * (decompression_settings.h:211-232, track_writer.h:170-186), rounding none, looping as_compressed,
 * layout QVV48, exact math. */
ACLB200_API void aclb200_default_options(aclb200_options* options);

/* Replaces make_decompression_context (decompress.h:205-209): binds a context to CUDA device `device`. */
ACLB200_API aclb200_status aclb200_create(int device, aclb200_context** out_context);
ACLB200_API void aclb200_destroy(aclb200_context* context);
/* Text of the last error raised on this context (never NULL). */
ACLB200_API const char* aclb200_last_error(const aclb200_context* context);

/* Replaces decompression_context::initialize(const compressed_tracks&) (decompress.h:90-101,
 * decompress.impl.h:66-83) for `num_clips` clips at once: validates every blob exactly like
 * compressed_tracks::is_valid(check_hash) + is_version_supported (v02_00_00 .. v02_01_00), copies the blobs to device memory (>= 64 bytes of tail slack for the `_unsafe` unaligned reads,
 * compress.transform.impl.h:387-396) and builds the acceleration index. Synchronous; the host blobs may be
 * freed when it returns. `out_failed_clip` (optional) receives the index of the first rejected clip.
 * A clip bound to a streaming database (compressed_tracks::has_database, what acl::build_database returns) is accepted and decodes from
 * the key frames that stay resident in the clip: what decompression_context<settings with database support>::initialize(tracks) gives
 * with no database bound, or with a database none of whose tiers is streamed in (decompress.impl.h:67-83, decompression.transform.h:
 * 262-265). Streaming the medium / low importance tiers in is not implemented. */
ACLB200_API aclb200_status aclb200_upload_clips(aclb200_context* context, const void* const* blobs, const uint32_t* sizes, uint32_t num_clips,
	uint32_t check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip);

/* Same, for clips stored back to back in one host buffer: clip i is buffer[offsets[i] .. offsets[i] + sizes[i]). */
ACLB200_API aclb200_status aclb200_upload_clips_packed(aclb200_context* context, const void* buffer, const uint64_t* offsets, const uint32_t* sizes,
	uint32_t num_clips, uint32_t check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip);

ACLB200_API void aclb200_release_clipset(aclb200_context* context, aclb200_clipset* clipset);
ACLB200_API aclb200_status aclb200_clipset_get_info(const aclb200_clipset* clipset, aclb200_clipset_info* out_info);
/* compressed_tracks accessors (compressed_tracks.h:60-140) */
ACLB200_API aclb200_status aclb200_clipset_get_clip_info(const aclb200_clipset* clipset, uint32_t clip, aclb200_clip_info* out_info);

/* ---- Streaming databases: acl::compressed_database + acl::database_context (decompression/database/database.h) ----
 * A clip built with acl::build_database keeps its most important key frames; the rest sit in a compressed_database, split into a medium
 * and a low importance tier of fixed-size chunks. Once its clip set is bound to the database, a clip decodes from whatever key frames
 * of the tiers are streamed in, exactly as a decompression_context initialised with a database_context does.
 *
 * Ordering: stream_in / stream_out enqueue their device work on `stream`. A decode enqueued on the same stream after the call sees the
 * new tier state; one enqueued before it does not. Work on another stream must wait for an event recorded after the call, as for every
 * other call of this library. A database must outlive the clip sets bound to it and the launches that read it. */

/* acl::quality_tier (core/quality_tier.h): the tiers a database stores */
enum { ACLB200_TIER_MEDIUM = 1, ACLB200_TIER_LOW = 2 };

typedef struct aclb200_database_info
{
	uint32_t num_chunks[2];			/* compressed_database::get_num_chunks(medium / low) */
	uint32_t bulk_data_size[2];		/* get_bulk_data_size(medium / low) */
	uint32_t max_chunk_size;		/* get_max_chunk_size() */
	uint32_t num_clips;				/* get_num_clips() */
	uint32_t num_segments;			/* get_num_segments() */
	uint32_t is_bulk_data_inline;	/* is_bulk_data_inline() */
	uint32_t hash;					/* get_hash() */
	uint32_t size;					/* get_size() */
} aclb200_database_info;

/* compressed_database::is_valid(check_hash) + the version check (core/impl/compressed_database.impl.h:142-162), plus bounds checks of
 * every chunk description, clip metadata entry and runtime segment header offset. A corrupt database fails with
 * ACLB200_ERR_INVALID_CLIP. The blob is copied: the caller may free it afterwards. Nothing is streamed in yet. */
ACLB200_API aclb200_status aclb200_upload_database(aclb200_context* context, const void* blob, uint32_t size, uint32_t check_hash,
	aclb200_database** out_database);
/* Waits for the device, then frees the database. */
ACLB200_API void aclb200_release_database(aclb200_context* context, aclb200_database* database);
ACLB200_API aclb200_status aclb200_database_get_info(const aclb200_database* database, aclb200_database_info* out_info);
/* Number of chunks of `tier` streamed in; database_context::is_streamed_in(tier) is loaded == num_chunks (database.impl.h:407-423). */
ACLB200_API aclb200_status aclb200_database_get_loaded_chunks(const aclb200_database* database, uint32_t tier, uint32_t* out_loaded_chunks);
/* database_context::stream_in(tier, num_chunks) (database.impl.h:443-523): picks the same chunk range (up to num_chunks chunks after
 * the last loaded one), copies it to the device and publishes the tier metadata of every segment in those chunks. `host_bulk_data` holds
 * the tier's whole bulk data (get_bulk_data_size(tier) bytes), or is NULL to use the bulk data inline in the database blob. Returns
 * once the host bytes have been read; *out_num_chunks (may be NULL) receives the number of chunks streamed (0: nothing left to do).
 * A tier with no chunks is an invalid argument. */
ACLB200_API aclb200_status aclb200_database_stream_in(aclb200_context* context, aclb200_database* database, uint32_t tier, uint32_t num_chunks,
	const void* host_bulk_data, uint32_t* out_num_chunks, void* stream);
/* database_context::stream_out(tier, num_chunks) (database.impl.h:525-637): unpublishes the first loaded chunks; the tier buffer is freed,
 * in stream order, with its last chunk. */
ACLB200_API aclb200_status aclb200_database_stream_out(aclb200_context* context, aclb200_database* database, uint32_t tier, uint32_t num_chunks,
	uint32_t* out_num_chunks, void* stream);
/* decompression_context::initialize(tracks, database) (decompress.impl.h:85-110) for every clip of the set: each clip bound to a database
 * (compressed_tracks::has_database) must be contained in `database`, else the call fails with ACLB200_ERR_INVALID_CLIP, names the first
 * such clip in *out_failed_clip and leaves the binding as it was. Clips without a database are unaffected. NULL unbinds. */
ACLB200_API aclb200_status aclb200_clipset_bind_database(aclb200_context* context, aclb200_clipset* clipset, const aclb200_database* database,
	uint32_t* out_failed_clip);

/* Replaces seek() + decompress_tracks(writer) (decompress.h:147-166; seek_v0 + decompress_tracks_v0,
 * decompression.transform.h:206-563,1526-1737) for `num_requests` requests in one fused kernel.
 * `d_requests` and `d_out` are device pointers; pose r starts at d_out + r * pose_stride_bytes and holds
 * one bone every 48 or 40 bytes (options->output_layout). Sub-tracks whose default mode is `skipped` are not
 * written. Transform clip sets only. */
ACLB200_API aclb200_status aclb200_decompress_tracks(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, void* d_out, void* stream);

/* Replaces seek() + decompress_track(track_index, writer) (decompress.h:168-172; decompress_track_v0,
 * decompression.transform.h:1753-2050): request r decodes bone d_track_indices[r] only and writes ONE bone
 * (48 / 40 bytes) at d_out + r * bone size. */
ACLB200_API aclb200_status aclb200_decompress_track(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, const uint32_t* d_track_indices, uint32_t num_requests,
	const aclb200_options* options, void* d_out, void* stream);

/* Scalar clip sets (float1f..float4f, vector4f): seek_v0 + decompress_tracks_v0 of decompression.scalar.h:181-481.
 * Request r writes num_tracks rows of `components` floats (write_float1..4 / write_vector4) at
 * d_out + r * pose_stride_bytes (0 = max_tracks * components * 4). Every float is written with one 4 byte store: d_out and
 * pose_stride_bytes must be multiples of 4, else the call fails with ACLB200_ERR_INVALID_ARGUMENT and launches nothing
 * (aclb200_decompress_tracks_host and aclb200_decompress_all_samples refuse such a stride the same way). */
ACLB200_API aclb200_status aclb200_scalar_decompress_tracks(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, void* d_out, void* stream);

/* decompress_track_v0 of decompression.scalar.h:483-705: one track per request, `components` floats each, at
 * d_out + r * components * 4. d_out must be a multiple of 4, else the call fails with ACLB200_ERR_INVALID_ARGUMENT and launches
 * nothing. */
ACLB200_API aclb200_status aclb200_scalar_decompress_track(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, const uint32_t* d_track_indices, uint32_t num_requests,
	const aclb200_options* options, void* d_out, void* stream);

/* Host-buffer convenience over aclb200_decompress_tracks / aclb200_scalar_decompress_tracks: copies `num_requests`
 * requests from host memory, decodes, copies the poses back to `out` (host) and waits. This is the call the C++
 * header shim uses to replay results into a host-side track_writer. Pinned host memory makes the copies faster
 * but is not required. options->d_request_policies, when given, stays a device array of num_requests pairs: request r
 * reads pair r whichever chunk decodes it. */
ACLB200_API aclb200_status aclb200_decompress_tracks_host(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* requests, uint32_t num_requests, const aclb200_options* options, void* out, size_t out_bytes);

/* ---- SURVEY 8(f1) / 8(f3): the nearest callers of the decode path, on the device (acl_b200/csrc/error_metric.cu) ---------------- */

/* acl::track_error (compression/track_error.h:48-62) + what the measurement met on the way */
typedef struct aclb200_track_error
{
	uint32_t index;					/* track with the worst error (0xFFFFFFFF when nothing was measured) */
	float    error;
	float    sample_time;
	uint32_t flags;					/* ACLB200_ERROR_FLAG_* */
} aclb200_track_error;

/* acl::itransform_error_metric implementations (compression/transform_error_metrics.h) */
enum
{
	ACLB200_METRIC_QVVF = 0,				/* qvvf_transform_error_metric (:281-385), and additive_qvvf_transform_error_metric<format> (:470-526) for the
											 * jobs that carry an additive_format */
	ACLB200_METRIC_QVVF_MATRIX3X4F = 1		/* qvvf_matrix3x4f_transform_error_metric (:389-464): transforms as 3x4 matrices (for rigs with shear);
											 * every operation is IEEE exact: bit-identical to the reference on any CPU */
};

enum
{
	ACLB200_ERROR_FLAG_NEGATIVE_SCALE = 1,		/* informational: a negative scale took rtm::qvv_mul through its matrix branch (qvvf.h:320-345) somewhere */
	ACLB200_ERROR_FLAG_INVALID_SKELETON = 2,	/* a parent index does not precede its child (the reference reads an unwritten transform there):
												 * the bone was treated as a root */
	ACLB200_ERROR_FLAG_WRAP_CLIP_CYCLE = 4,		/* aclb200_extract_root_motion: a request crossed a loop boundary of a clip compressed with the
												 * wrap policy, whose motion from its last sample back to its first is missing (see there) */
	ACLB200_ERROR_FLAG_INVALID_MIRROR = 8		/* the mirror decodes and aclb200_mirror_poses: a mirror table entry names a row out of range or a
												 * row that does not name it back; that row took its own transform (see aclb200_mirror_entry) */
};

/* One clip to measure == one `calculate_compression_error(allocator, raw_tracks, context, error_metric)` call of the reference
 * (compression/track_error.h:64-121). The raw clip arrives already sampled: pose s of the job is what
 * `raw_tracks.sample_tracks(min(s / sample_rate, duration), rounding, writer)` writes (track_error.impl.h:337-338,504-507), where rounding is
 * nearest, or none when the compressed clip has stripped key frames (:556-559). */
typedef struct aclb200_error_job
{
	uint32_t clip;					/* index into the clip set */
	uint32_t num_samples;			/* raw_tracks.get_num_samples_per_track() */
	float    sample_rate;			/* raw_tracks.get_sample_rate() */
	float    duration;				/* raw_tracks.get_finite_duration() */
	uint32_t num_tracks;			/* raw_tracks.get_num_tracks() */
	uint32_t skeleton_offset;		/* first entry of this clip's skeleton in d_parent_indices / d_shell_distances / d_output_indices */
	uint64_t first_raw_pose;		/* pose index of sample 0 in d_raw_poses */
	uint32_t additive_format;		/* acl::additive_clip_format8 (core/additive_utils.h:42-66): 0 none, 1 relative, 2 additive0, 3 additive1 */
	uint32_t error_metric;			/* ACLB200_METRIC_* (transform clip sets) */
	uint64_t first_base_pose;		/* additive jobs: pose index of sample 0 in d_base_poses */
} aclb200_error_job;

/* Replaces calculate_compression_error (compression/impl/track_error.impl.h:400-571: calculate_transform_track_error :225-392 with the
 * qvvf_transform_error_metric of compression/transform_error_metrics.h:281-385, calculate_scalar_track_error :166-223) for `num_jobs` clips:
 * every sample of every clip is decoded on the device (decompress_tracks, rounding as above, `options` = the settings / writer of the context
 * the reference would be handed: pass the bind pose as constant or variable defaults), taken to object space and compared with the raw pose.
 *   jobs              HOST array
 *   d_raw_poses       device: pose p at p * pose_stride_bytes (options, 0 = max_tracks * 48): rtm::qvvf per bone (transform clip sets),
 *                     `components` floats per track (scalar clip sets: the layout aclb200_scalar_decompress_tracks writes)
 *   d_parent_indices  device: track_desc_transformf::parent_index per track (0xFFFFFFFF = root; a parent precedes its children),
 *   d_shell_distances device: track_desc_transformf::shell_distance per track; both unused (NULL) for scalar clip sets
 *   d_output_indices  device, optional: track_desc::output_index per raw track (0xFFFFFFFF = stripped from the compressed clip: the raw
 *                     value stands in, track_error.impl.h:522-532); NULL = every raw track i is output i
 *   d_base_poses      device, optional: the additive base of the jobs whose additive_format is not 0 (the calculate_compression_error
 *                     overload with additive_base_tracks, track_error.impl.h:573-680, + additive_qvvf_transform_error_metric<format>,
 *                     transform_error_metrics.h:470-526): pose s of a job is `additive_base_tracks.sample_tracks(t_base(s), rounding, writer)`
 *                     with t_base = (t / duration) * base_duration, or 0 when the base has one sample (:352-356); it is applied to the raw
 *                     and to the decoded pose with acl::apply_additive_to_base (core/additive_utils.h:147-157) before the hierarchy walk
 *   d_out_errors      device: one aclb200_track_error per job
 *   d_out_error_matrix device, optional: the error of every bone of every pose, row (poses of the earlier jobs + s) of
 *                     pose_stride_bytes / 48 floats (= max_tracks by default; scalar clip sets: tracks per row)
 * rtm::quat_normalize's rsqrtss estimate is CPU specific: errors agree with a given CPU's
 * within 5e-5 on poses tens of units across, not bit for bit (see error_metric.cu). Asynchronous on `stream`; uses scratch owned by the context.
 * That scratch is shared with aclb200_decompress_all_samples: each call's work on `stream` waits for the previous such call on the
 * context to finish reading it, on whatever stream that call ran, so calls on different streams run one after the other on the device
 * (never at the same time), and a call that has to grow the scratch first waits on the host for that previous call.
 * A clip set whose bound database has chunks streamed in is refused with ACLB200_ERR_UNSUPPORTED: these measurements never ignore tiers. */
ACLB200_API aclb200_status aclb200_calculate_compression_error(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
	uint32_t num_jobs, const void* d_raw_poses, const uint32_t* d_parent_indices, const float* d_shell_distances,
	const uint32_t* d_output_indices, const void* d_base_poses, const aclb200_options* options, aclb200_track_error* d_out_errors,
	float* d_out_error_matrix, void* stream);

/* The sampling loop of acl::convert_track_list(allocator, const compressed_tracks&, track_array&) (compression/convert.h,
 * compression/impl/convert.impl.h:146-232) and of the error measurement above: EVERY sample of every listed clip in one launch sequence.
 * Job j contributes num_samples poses, sample i sought at min(i / sample_rate, duration) with options->rounding_policy (the reference
 * uses `nearest` "to land directly on a sample") and decoded like aclb200_decompress_tracks / aclb200_scalar_decompress_tracks would:
 * the poses of the jobs follow one another in d_out (pose stride and layout from `options`). Only clip, num_samples, sample_rate and
 * duration of a job are read. jobs is a HOST array; asynchronous on `stream`; uses scratch owned by the context, ordered after the
 * previous call that used it on any stream (see aclb200_calculate_compression_error).
 * ACLB200_ERR_UNSUPPORTED on a clip set whose bound database has chunks streamed in. */
ACLB200_API aclb200_status aclb200_decompress_all_samples(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
	uint32_t num_jobs, const aclb200_options* options, void* d_out, void* stream);

/* Decoded poses held per chunk of clips by aclb200_calculate_compression_error (default 1 GiB). */
ACLB200_API aclb200_status aclb200_set_error_chunk_bytes(aclb200_context* context, uint64_t bytes);

/* Replaces qvvf_transform_error_metric::local_to_object_space (compression/transform_error_metrics.h:289-310: obj[i] =
 * qvv_normalize(qvv_mul(local[i], obj[parent[i]])), roots copied) for `num_poses` poses of one skeleton: rtm::qvvf rows in, rtm::qvvf rows
 * out (48 byte bones, pose_stride_bytes 0 = num_tracks * 48; the two buffers may be the same). d_out_flags (optional, device uint32):
 * ACLB200_ERROR_FLAG_* met on the way. */
ACLB200_API aclb200_status aclb200_local_to_object_space(aclb200_context* context, const void* d_local_poses, void* d_object_poses, uint64_t num_poses,
	uint32_t num_tracks, uint64_t pose_stride_bytes, const uint32_t* d_parent_indices, uint32_t* d_out_flags, void* stream);

/* What aclb200_decompress_tracks_object_space writes per bone (48 bytes either way) */
enum
{
	ACLB200_OBJECT_QVVF = 0,		/* rtm::qvvf: rotation xyzw, translation xyz + 0, scale xyz + 0 (what aclb200_local_to_object_space writes) */
	ACLB200_OBJECT_MATRIX3X4F = 1	/* rtm::matrix3x4f without its constant w lanes: x_axis xyz, y_axis xyz, z_axis xyz, w_axis xyz */
};

/* aclb200_decompress_tracks followed by the hierarchy walk, in one kernel: the local poses never leave shared memory. Request r computes
 * what aclb200_decompress_tracks computes for it (same options, rounding, looping, per request policies, default modes and bind pose;
 * a clip set whose bound database has chunks streamed in decodes from them) and takes the pose to object space with its clip's skeleton:
 *   ACLB200_OBJECT_QVVF       qvvf_transform_error_metric::local_to_object_space (transform_error_metrics.h:289-310):
 *                             obj = qvv_normalize(qvv_mul(local, obj[parent])), roots copied; byte for byte what
 *                             aclb200_local_to_object_space writes for the decoded pose
 *   ACLB200_OBJECT_MATRIX3X4F convert_transforms (matrix_from_qvv) + local_to_object_space of qvvf_matrix3x4f_transform_error_metric
 *                             (:397-436): obj = matrix_mul(local, obj[parent]), roots copied; bit-identical to the reference on any CPU
 * Every operation is IEEE and unfused; ACLB200_MATH_FAST is accepted and runs the exact decode.
 *   d_parent_indices    device: parent of each bone (0xFFFFFFFF = root); clip c's skeleton starts at d_parent_indices + d_skeleton_offsets[c]
 *   d_skeleton_offsets  device u32[num_clips], or NULL: every clip uses the skeleton at offset 0
 *   d_out               pose r at d_out + r * options->pose_stride_bytes (0 = max_tracks * 48), 48 bytes per bone; stride and alignment
 *                       as aclb200_decompress_tracks requires for ACLB200_LAYOUT_QVV48. A request with an invalid clip index writes
 *                       nothing, and no byte past a clip's num_tracks * 48 is written.
 *   d_out_flags         device uint32, optional: cleared, then ACLB200_ERROR_FLAG_* met on the way OR-ed in, as aclb200_local_to_object_space
 *                       does (a parent that does not precede its child is reported and its bone treated as a root)
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, writing nothing: skip masks (options->skip_mask, d_skip_track_mask) or a `skipped` default mode
 * (an object transform needs every sub-track of its parents), an output layout other than QVV48, an unknown object_kind, NULL parents, a
 * scalar clip set. ACLB200_ERR_UNSUPPORTED when one pose does not fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_object_space(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* acl::additive_clip_format8 (core/additive_utils.h:42-66): how an additive clip applies to its base */
enum { ACLB200_ADDITIVE_NONE = 0, ACLB200_ADDITIVE_RELATIVE = 1, ACLB200_ADDITIVE_ADDITIVE0 = 2, ACLB200_ADDITIVE_ADDITIVE1 = 3 };

/* One layered pose: an additive clip sampled on top of a base clip. Both clips live in the same clip set; the two sample times are
 * independent (keeping them in sync is the caller's business). */
typedef struct aclb200_additive_request
{
	aclb200_request base;			/* the base clip and its sample time */
	aclb200_request additive;		/* the additive clip and its sample time */
} aclb200_additive_request;

/* decompress base + decompress additive + acl::apply_additive_to_base (core/additive_utils.h:152-162) per bone, in one kernel: neither
 * pose leaves shared memory. For pair r:
 *   base pose      what aclb200_decompress_tracks computes for requests[r].base with `options` (rounding, looping, per request policies
 *                  -- d_request_policies[r] applies to both halves --, per track rounding, normalisation, default modes and bind pose, a
 *                  bound database's streamed tiers)
 *   additive pose  the same for requests[r].additive, except that its default sub-tracks take the acl::track_writer defaults
 *                  (track_writer.h:160-176): identity rotation, zero translation, the clip's own default scale (0 for additive1 clips)
 *   format         d_clip_additive_formats[requests[r].additive.clip] (a byte above 3 reads as none) when that pointer is not NULL,
 *                  else additive_format: none = the additive pose, relative = rtm::qvv_mul(additive, base) (its matrix branch for
 *                  negative scales included), additive0 / additive1 = transform_add0 / transform_add1 (additive_utils.h:131-145)
 *   d_out          d_parent_indices == NULL: the combined local pose in options->output_layout at d_out + r * options->pose_stride_bytes
 *                  (0 = max_tracks * bone size). d_parent_indices given: the combined pose goes through the hierarchy walk of
 *                  aclb200_decompress_tracks_object_space with the skeleton d_parent_indices + d_skeleton_offsets[requests[r].base.clip]
 *                  (d_skeleton_offsets NULL: 0) and leaves as object_kind rows (QVV48 only).
 *                  A pair with an invalid clip index on either side, or with clips of different track counts, writes nothing; no byte
 *                  past a clip's num_tracks bones is written.
 *   d_out_flags    device uint32, optional: cleared, then ACLB200_ERROR_FLAG_NEGATIVE_SCALE (a relative bone or the walk took qvv_mul's
 *                  matrix branch) and ACLB200_ERROR_FLAG_INVALID_SKELETON OR-ed in
 * Every operation is IEEE and unfused; ACLB200_MATH_FAST is accepted and runs the exact decode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, writing nothing: skip masks, a `skipped` default mode, additive_format > 3, a scalar clip
 * set, an output that breaks the alignment rules of aclb200_decompress_tracks, and with parents an unknown object_kind or QVV40.
 * ACLB200_ERR_UNSUPPORTED when the two poses of a pair do not fit in one block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_additive(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* acl::apply_additive_to_base(additive_format, base, additive) on every bone of num_poses poses of rtm::qvvf rows (48 byte bones, 16 byte
 * aligned; pose p of each buffer at p * pose_stride_bytes, 0 = num_tracks * 48): for a base pose that does not come from one clip (a
 * blend). d_out may be either input. The translation and scale w lanes are written as 0. d_out_flags as aclb200_decompress_tracks_additive.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT: NULL pointers, additive_format > 3, misaligned rows. */
ACLB200_API aclb200_status aclb200_apply_additive_to_base(aclb200_context* context, const void* d_base_poses, const void* d_additive_poses,
	void* d_out, uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride_bytes, uint32_t additive_format,
	uint32_t* d_out_flags, void* stream);

/* One blended pose: two clips of the same clip set, each at its own sample time (a crossfade, or a blend of walk and run) */
typedef struct aclb200_blend_request
{
	aclb200_request from;			/* weight 0 gives this pose */
	aclb200_request to;				/* weight 1 gives this pose (or its hemisphere-flipped rotation) */
} aclb200_blend_request;

/* decompress from + decompress to + rtm::qvv_lerp(from, to, w) (rtm/qvvf.h:439-445) per bone, in one kernel: neither pose leaves shared
 * memory. For pair r:
 *   both poses     what aclb200_decompress_tracks computes for requests[r].from and requests[r].to with `options` (rounding, looping, per
 *                  request policies -- d_request_policies[r] applies to both halves --, per track rounding, normalisation, default modes and
 *                  bind pose, a bound database's streamed tiers). Neither half takes the track_writer defaults: both are full poses.
 *   w              d_weights[r] (device float[num_requests]) when d_weights is not NULL, else `weight`; used as given, no clamp: below 0 and
 *                  above 1 extrapolate, as rtm does
 *   blend          rtm::quat_lerp's SSE4.1 path: dot = (x x' + y y') + (z z' + w w'); `to`'s rotation is negated when the SIGN BIT of dot is
 *                  set (dot == -0.0 included); q = (s - w s) + w to per lane, then quat_normalize with an IEEE 1 / sqrt (the reference's
 *                  rsqrtss + 2 Newton-Raphson steps is CPU specific: rotations agree within 1e-6). Translations and scales are
 *                  rtm::vector_lerp: (s - s w) + e w, bit-identical to the reference. The translation and scale w lanes are written as 0.
 *   d_out          d_parent_indices == NULL: the blended local pose in options->output_layout at d_out + r * options->pose_stride_bytes
 *                  (0 = max_tracks * bone size). d_parent_indices given: the blended local pose goes through the hierarchy walk of
 *                  aclb200_decompress_tracks_object_space with the skeleton d_parent_indices + d_skeleton_offsets[requests[r].from.clip]
 *                  (d_skeleton_offsets NULL: 0) and leaves as object_kind rows (QVV48 only): blend in local space, then to object space.
 *                  A pair with an invalid clip index on either side, or with clips of different track counts, writes nothing; no byte
 *                  past a clip's num_tracks bones is written.
 *   d_out_flags    device uint32, optional: cleared, then the walk's ACLB200_ERROR_FLAG_NEGATIVE_SCALE and ACLB200_ERROR_FLAG_INVALID_SKELETON
 *                  OR-ed in (the blend itself raises none)
 * Every operation is IEEE and unfused; ACLB200_MATH_FAST is accepted and runs the exact decode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, writing nothing: skip masks, a `skipped` default mode, a scalar clip set, an output that breaks
 * the alignment rules of aclb200_decompress_tracks, and with parents an unknown object_kind or QVV40.
 * ACLB200_ERR_UNSUPPORTED when the two poses of a pair do not fit in one block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_blend(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	float weight, const float* d_weights,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* rtm::qvv_lerp(from, to, w) as aclb200_decompress_tracks_blend computes it, on every bone of num_poses poses of rtm::qvvf rows (48 byte
 * bones, 16 byte aligned; pose p of each buffer at p * pose_stride_bytes, 0 = num_tracks * 48), w = d_weights[p] (device float[num_poses])
 * or `weight` when d_weights is NULL: for poses already on the device, such as a chain of blends (a 2D blend space is lerps of lerps) or a
 * decoded pose and a pose from elsewhere. d_out may be either input. The translation and scale w lanes are written as 0.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT: NULL pointers, misaligned rows. */
ACLB200_API aclb200_status aclb200_blend_poses(aclb200_context* context, const void* d_from_poses, const void* d_to_poses, void* d_out,
	uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride_bytes, float weight, const float* d_weights, void* stream);

/* Skinning matrices: the pose of aclb200_decompress_tracks_object_space, _additive or _blend taken through the ACLB200_OBJECT_MATRIX3X4F
 * walk (convert_transforms + local_to_object_space of qvvf_matrix3x4f_transform_error_metric, transform_error_metrics.h:397-436; never the
 * qvvf walk, so no quat_normalize), then per bone
 *     skin[b] = rtm::matrix_mul(inverse_bind[b], object[b])       (matrix3x4f.h:298-321, rtm's row vector order)
 * in one kernel: the local and object rows never leave shared memory. Every step is an IEEE multiply or add in the reference's order, so
 * wherever the route's matrix rows are bit-identical to the reference, so are its skinning rows.
 *   d_inverse_bind   device, 16 byte aligned: one rtm::matrix3x4f per skeleton entry, in parallel with d_parent_indices (clip c, bone b reads
 *                    d_inverse_bind + 12 * (d_skeleton_offsets[c] + b)), as the xyz lanes of x_axis, y_axis, z_axis, w_axis (the 12 floats
 *                    ACLB200_OBJECT_MATRIX3X4F writes). A bone that is not skinned takes the identity.
 *   d_out            48 bytes per bone, three float4 rows: row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]) of skin, so that component
 *                    c of rtm::matrix_mul_point3(p, skin) is dot(row c, (p, 1)): what a skinning shader reads. Stride, alignment, invalid
 *                    clips and pairs, and bytes past num_tracks * 48 as the entry point each call mirrors.
 *   d_out_flags      as that entry point: ACLB200_ERROR_FLAG_INVALID_SKELETON from the walk, ACLB200_ERROR_FLAG_NEGATIVE_SCALE from an
 *                    additive `relative` bone that took qvv_mul's matrix branch (the matrix walk itself has no branch)
 * The skeleton and the inverse binds are those of the base clip (additive) or of the from clip (blend).
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, writing nothing: NULL parents or inverse binds, a d_inverse_bind that is not 16 byte aligned,
 * skip masks or a `skipped` default mode, an output layout other than QVV48, a scalar clip set, additive_format > 3, an output that breaks
 * the alignment rules of aclb200_decompress_tracks. ACLB200_ERR_UNSUPPORTED when a pose (or a pair) does not fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);
ACLB200_API aclb200_status aclb200_decompress_tracks_additive_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);
ACLB200_API aclb200_status aclb200_decompress_tracks_blend_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	float weight, const float* d_weights,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* What a layer does to the running pose of its stack (aclb200_decompress_tracks_layered) */
enum { ACLB200_LAYER_OFF = 0, ACLB200_LAYER_BLEND = 1, ACLB200_LAYER_ADDITIVE = 2 };

/* One layer of a layered pose: a clip of the clip set at its own sample time, and what it does to the poses below it */
typedef struct aclb200_layer
{
	aclb200_request pose;			/* this layer's clip and sample time */
	uint32_t op;					/* ACLB200_LAYER_* */
	float    weight;				/* BLEND: the rtm::qvv_lerp weight, used as given (no clamp); ADDITIVE: ignored by
									   aclb200_decompress_tracks_layered, the weight of the delta in _layered_masked; ignored otherwise */
} aclb200_layer;

/* A pose graph of up to eight clips per pose in one kernel: every layer is decoded, and the layers are folded into the running pose in
 * index order in shared memory; only the result leaves. Pose r owns the layers d_layers[r * num_layers + i], 1 <= num_layers <= 8:
 *   base           the first layer whose op is not OFF, decoded exactly as aclb200_decompress_tracks decodes its request under `options`
 *                  (its op and weight are ignored). The running pose starts as the base.
 *   later layers   in index order:
 *                    OFF       not sought, not decoded, not read (its clip and time may be anything, no key frame traffic): stacks of
 *                              different depths share one launch
 *                    BLEND     decoded as a full pose (as either half of aclb200_decompress_tracks_blend), then
 *                              running = rtm::qvv_lerp(running, layer, weight), computed as aclb200_decompress_tracks_blend computes it
 *                    ADDITIVE  decoded with the acl::track_writer defaults (as the additive half of aclb200_decompress_tracks_additive),
 *                              then running = acl::apply_additive_to_base(format, running, layer), format = d_clip_additive_formats[the
 *                              layer's clip] (a byte above 3 reads as none) when that pointer is not NULL, else additive_format
 *   policies       d_request_policies[r] (options) applies to every layer of pose r
 *   d_out          d_parent_indices == NULL: the running pose in options->output_layout (QVV48 or QVV40) at d_out + r * pose_stride
 *                  (options->pose_stride_bytes, 0 = max_tracks * bone size). d_parent_indices given: the hierarchy walk of
 *                  aclb200_decompress_tracks_object_space with the skeleton of the BASE layer's clip c (d_parent_indices +
 *                  d_skeleton_offsets[c], d_skeleton_offsets NULL: 0), object_kind rows (QVV48 only).
 *                  Pose r writes nothing when every layer is OFF, when a layer that is not OFF names an invalid clip or a clip whose track
 *                  count differs from the base's, or when any layer's op is above 2. No byte past the base clip's num_tracks bones is written.
 *   d_out_flags    device uint32, optional: cleared, then ACLB200_ERROR_FLAG_NEGATIVE_SCALE (a relative layer took qvv_mul's matrix branch,
 *                  or the walk did) and ACLB200_ERROR_FLAG_INVALID_SKELETON OR-ed in
 * Blend-space weights: the stack [clip 0 as base, clip 1 BLEND w_1, ..., clip n BLEND w_n] gives the normalised blend
 * sum_i a_i clip_i (a_0 + ... + a_n = 1) of the lerps' translations and scales with the step weights
 *     w_i = a_i / (a_0 + a_1 + ... + a_i)
 * (each step's lerp keeps the ratios of the clips before it); additive layers then go on top.
 * Every operation is IEEE and unfused; ACLB200_MATH_FAST is accepted and runs the exact decode.
 * Refused, writing nothing and leaving *d_out_flags untouched: ACLB200_ERR_INVALID_ARGUMENT for num_layers 0 or above 8, num_poses *
 * num_layers above 2^32 - 1, skip masks or a `skipped` default mode, additive_format > 3, a scalar clip set, an output that breaks the
 * alignment rules of aclb200_decompress_tracks, and with parents an unknown object_kind or QVV40. ACLB200_ERR_UNSUPPORTED when
 * num_layers poses of the widest clip do not fit in one block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_layered(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The skinning rows of the layered pose: aclb200_decompress_tracks_layered's running pose through the matrix walk and the skinning step
 * of aclb200_decompress_tracks_skinning, with the base layer's skeleton and inverse binds (d_inverse_bind + 12 * d_skeleton_offsets[base
 * clip]). Refusals as aclb200_decompress_tracks_layered, plus NULL parents and NULL or misaligned inverse binds. */
ACLB200_API aclb200_status aclb200_decompress_tracks_layered_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The mask index of a layer without a bone mask (aclb200_decompress_tracks_layered_masked) */
#define ACLB200_LAYER_NO_MASK 0xFFFFFFFFu

/* Masked layer stacks: aclb200_decompress_tracks_layered with a per-bone weight mask on any layer (partial-body layers: an upper-body
 * aim over lower-body locomotion, a wave on one arm, a feathered spine) and ADDITIVE layers that take their weight, in one kernel.
 * Everything not listed here is as aclb200_decompress_tracks_layered (and _layered_skinning): base, OFF layers, decode, formats,
 * policies, d_out, object kinds, skeletons, inverse binds, d_out_flags, database tiers, ACLB200_MATH_FAST, the shared memory limits.
 *   d_layer_masks  device uint32[num_poses * num_layers] or NULL (no layer has a mask): d_layer_masks[r * num_layers + i] is the mask
 *                  index of layer i of pose r, ACLB200_LAYER_NO_MASK for none. The mask index of an OFF layer or of the base is not read.
 *   d_bone_masks   device float[num_masks * mask_stride], 4 byte aligned: mask m is d_bone_masks[m * mask_stride + b], one float per bone b
 *                  of the BASE clip's skeleton (mask_stride 0: the clip set's max_tracks). Masks belong to a rig: a launch that mixes rigs
 *                  names the right mask per layer.
 *   weight at b    w_b = weight * mask[b] (one IEEE multiply), or weight for a layer without a mask. A mask value of +0 or -0 leaves
 *                  bone b untouched, byte for byte: the bones outside a mask are those of the stack without the layer.
 *   BLEND          running = rtm::qvv_lerp(running, layer, w_b) as aclb200_decompress_tracks_blend computes it; w_b used as given.
 *   ADDITIVE       w_b == 1: running = acl::apply_additive_to_base(format, running, layer), what _layered computes. Otherwise
 *                  running = acl::apply_additive_to_base(format, running, rtm::qvv_lerp(identity, layer, w_b)), identity = the track_writer
 *                  default pose the layer is decoded with (identity rotation, zero translation, the clip's default scale: 1, or 0 for
 *                  additive1 clips), the identity of every format: w_b scales the additive delta. Weight 0 is applied (an identity
 *                  delta), a mask of 0 skips.
 *   writes nothing as aclb200_decompress_tracks_layered, and also when a BLEND or ADDITIVE layer above the base names a mask index at or
 *                  above num_masks (other than ACLB200_LAYER_NO_MASK).
 * Migration: with every ADDITIVE weight set to 1 and no masks (d_layer_masks NULL), the outputs equal aclb200_decompress_tracks_layered's
 * byte for byte.
 * Refused, writing nothing and leaving *d_out_flags untouched: what aclb200_decompress_tracks_layered (_layered_skinning) refuses, and
 * with d_layer_masks given: d_bone_masks NULL or not 4 byte aligned, num_masks 0 or above 2^29 - 1, a mask_stride below max_tracks,
 * num_masks * mask_stride above 2^32 - 1 (ACLB200_ERR_INVALID_ARGUMENT). */
ACLB200_API aclb200_status aclb200_decompress_tracks_layered_masked(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers,
	const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);
ACLB200_API aclb200_status aclb200_decompress_tracks_layered_masked_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers,
	const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options* options,
	uint32_t additive_format, const uint8_t* d_clip_additive_formats,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The bones per list of aclb200_decompress_bones, and an unused entry of a bone list */
#define ACLB200_MAX_QUERY_BONES 32
#define ACLB200_NO_BONE 0xFFFFFFFFu

/* Bone queries: chosen bones of each pose (attachment sockets, IK effectors and feet, motion matching features, the root), in one kernel
 * that decodes and walks only the ancestor chains of the requested bones and stores only the requested rows.
 *   bone lists      K = bones_per_list (1..ACLB200_MAX_QUERY_BONES); list l is d_bone_lists[l * K .. l * K + K - 1] (device). Request r
 *                   uses list d_request_lists[r] (device uint32[num_requests]), or list 0 for every request when d_request_lists is NULL.
 *                   A list may hold duplicates, any order and ACLB200_NO_BONE holes. A request whose list index is >= num_lists writes
 *                   nothing.
 *   d_out           entry j of request r's list at d_out + r * pose_stride + j * bone size; pose_stride = options->pose_stride_bytes, 0 =
 *                   K * bone size (48 bytes, or 40 for local QVV40 rows); alignment as aclb200_decompress_tracks requires for the layout.
 *                   An entry that is ACLB200_NO_BONE, or at or above its clip's num_tracks, leaves its row untouched (as
 *                   aclb200_decompress_track does with an invalid track index). A request with an invalid clip index writes nothing.
 *   local rows      d_parent_indices NULL: row j is row list[j] of what aclb200_decompress_tracks computes for the request with the same
 *                   options, in options->output_layout (QVV48 or QVV40), byte for byte. Only the listed bones are decoded, with
 *                   aclb200_decompress_tracks's arithmetic (not aclb200_decompress_track's normalisation).
 *   object rows     d_parent_indices given: row j is row list[j] of aclb200_decompress_tracks_object_space for the same request, options,
 *                   skeleton (d_parent_indices + d_skeleton_offsets[clip], d_skeleton_offsets NULL: 0) and object_kind
 *                   (ACLB200_OBJECT_QVVF or ACLB200_OBJECT_MATRIX3X4F; QVV48 only), byte for byte. Only the bones on the listed bones'
 *                   ancestor chains are decoded and walked. A parent that does not precede its child ends the chain and its bone is
 *                   treated as a root, as the whole walk does: the ancestor walk only ever moves to a lower bone index, so it ends on any
 *                   parent table.
 *   d_out_flags     device uint32, optional: cleared, then the ACLB200_ERROR_FLAG_* met on the walked bones OR-ed in. This can be fewer
 *                   bits than aclb200_decompress_tracks_object_space reports for the same poses: a mirrored bone or a bad parent outside
 *                   every chain is not walked.
 * As aclb200_decompress_tracks_object_space: per request and per track policies, default modes and variable defaults, a bound database's
 * streamed tiers; every operation IEEE and unfused, ACLB200_MATH_FAST accepted and runs the exact decode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, writing nothing and leaving *d_out_flags untouched: bones_per_list 0 or above 32, num_lists 0,
 * NULL d_bone_lists, skip masks or a `skipped` default mode, a scalar clip set, with parents an unknown object_kind or QVV40, a pose stride
 * below K * bone size, the alignment rules of aclb200_decompress_tracks. ACLB200_ERR_UNSUPPORTED when one pose of the widest clip does not
 * fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_bones(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list, const uint32_t* d_request_lists,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* One root motion request: how far the root moved between two playback times of one clip */
typedef struct aclb200_root_motion_request
{
	uint32_t clip;				/* index into the clip set */
	float    from_time;			/* playback time at the previous update, seconds */
	float    to_time;			/* playback time now */
	int32_t  cycles;			/* loop boundaries crossed from from_time to to_time: 0 none; k > 0 playback ran forward past the clip's end
								 * k times; k < 0 it ran backward past the start -k times */
} aclb200_root_motion_request;

/* The most loop boundaries one root motion request may cross */
#define ACLB200_MAX_ROOT_MOTION_CYCLES 256

/* Root motion: the root's displacement between the playback time of the previous update and the current one, across loop boundaries, in
 * one launch. It moves the character, not the pose. The reference's clamp policy exists for this use: "This makes it possible to extract
 * the total root motion by sampling at the full duration of the clip and at 0 seconds" (core/sample_looping_policy.h:47-55,
 * docs/handling_looping_playback.md:22).
 *   d_requests      device aclb200_root_motion_request[num_requests], 4 byte aligned (the alignment of its fields; no wider alignment is
 *                   assumed).
 *   root track      request r uses track d_root_tracks[clip] (device uint32[num_clips]), or track 0 when d_root_tracks is NULL.
 *   T(t)            the root track's row of aclb200_decompress_tracks for the request {clip, t} with the same options, in QVV48, read as an
 *                   rtm::qvvf. Every sample is taken with ACLB200_LOOP_CLAMP; times are clamped and rounded as aclb200_decompress_tracks
 *                   does (the batch rounding policy, d_per_track_rounding). D is the clip's clamp duration (num_samples - 1) / sample_rate:
 *                   T(D) is its last sample, T(0) its first.
 *   rel(a, b)       rtm::qvv_mul(T(b), rtm::qvv_inverse(T(a))) (qvvf.h:315-355 with both branches; the one argument qvv_inverse,
 *                   qvvf.h:389-395, whose vector_reciprocal is an IEEE division under SSE2, vector4f.h:1310). It is the delta with
 *                   T(b) = qvv_mul(rel(a, b), T(a)), in the root's frame at a: an engine accumulates it as M <- qvv_mul(delta, M).
 *   M               cycles == 0: rel(from, to), in either direction.
 *                   cycles = k > 0: M = rel(from, D); then k - 1 times M = qvv_mul(rel(0, D), M); then M = qvv_mul(rel(0, to), M).
 *                   cycles = k < 0: M = rel(from, 0); then -k - 1 times M = qvv_mul(rel(D, 0), M); then M = qvv_mul(rel(D, to), M).
 *                   The full cycle delta is computed once per request; nothing is normalised beyond what rtm's functions do.
 *   d_out           M of request r at d_out + r * 48 (16 byte aligned): rotation xyzw, translation xyz + 0, scale xyz + 0, the layout of
 *                   ACLB200_OBJECT_QVVF rows. options->pose_stride_bytes is not used. A request with an invalid clip index, a root track
 *                   at or beyond its clip's num_tracks or |cycles| > ACLB200_MAX_ROOT_MOTION_CYCLES leaves its row untouched.
 *   d_out_flags     device uint32, optional: cleared, then OR-ed in: ACLB200_ERROR_FLAG_NEGATIVE_SCALE when a qvv_mul took its matrix
 *                   branch (a mirrored root); ACLB200_ERROR_FLAG_WRAP_CLIP_CYCLE when a request that writes its row has cycles != 0 on a
 *                   clip compressed with the wrap policy (aclb200_clip_info::looping_policy). Such a clip has no sample at its end, so
 *                   the interval from its last sample back to its first contributes no motion: reported, not repaired.
 * As aclb200_decompress_bones: a bound database's streamed tiers are read, variable defaults and the batch and per track rounding policies
 * are honoured, ACLB200_MATH_FAST is accepted and runs the exact decode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing and leaving *d_out_flags untouched: NULL d_requests or d_out with
 * num_requests > 0, d_out not 16 byte aligned, output_layout other than QVV48, looping_policy other than ACLB200_LOOP_CLAMP, a non-NULL
 * d_request_policies (its looping byte would contradict the clamp rule), skip masks or a `skipped` default mode, a scalar clip set. */
ACLB200_API aclb200_status aclb200_extract_root_motion(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_root_motion_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const uint32_t* d_root_tracks, void* d_out, uint32_t* d_out_flags, void* stream);

/* One pose features request: the playback time of a character on one clip, and how its offsets reach beyond the clip's ends */
typedef struct aclb200_feature_request
{
	uint32_t clip;				/* index into the clip set */
	float    time;				/* the current playback time t, seconds */
	uint32_t looping;			/* ACLB200_FEATURE_CLAMP or ACLB200_FEATURE_LOOP */
} aclb200_feature_request;

/* aclb200_feature_request::looping: an offset time beyond the clip's ends is clamped, or wraps around into the next or previous cycle */
#define ACLB200_FEATURE_CLAMP 0u
#define ACLB200_FEATURE_LOOP 1u
/* The most time offsets of one aclb200_extract_pose_features launch */
#define ACLB200_MAX_FEATURE_OFFSETS 8

/* Pose features (motion matching): chosen bones of each request at up to eight time offsets, each in the character's frame at the request's
 * time, in one launch. For request r, offset s (S = num_offsets) and entry k of the request's bone list (K = bones_per_list):
 *   d_requests      device aclb200_feature_request[num_requests] (12 bytes each), 4 byte aligned.
 *   offsets         HOST float[num_offsets] in seconds (1..ACLB200_MAX_FEATURE_OFFSETS), copied into the launch: negative for the past, 0
 *                   for the current pose, positive for the predicted trajectory.
 *   bone lists      as aclb200_decompress_bones (d_bone_lists, num_lists, bones_per_list, d_request_lists).
 *   root track      d_root_tracks[clip] (device uint32[num_clips]), or track 0 when d_root_tracks is NULL. D is the clip's clamp duration,
 *                   as aclb200_extract_root_motion's.
 *   offset time     u = t + offsets[s] (one IEEE single add). ACLB200_FEATURE_CLAMP: c = 0, u' = u (the seek clamps u' as
 *                   aclb200_decompress_tracks does). ACLB200_FEATURE_LOOP: D == 0 gives c = 0, u' = 0; otherwise c = (int32) floorf(u / D)
 *                   and u' = u - float(c) * D, an IEEE divide, multiply and subtract, none fused.
 *   M_s             byte for byte the row aclb200_extract_root_motion writes for {clip, t, u', c} with the same options and root.
 *   T_s             the root track's local row at u': aclb200_decompress_tracks's QVV48 row with the clamp policy.
 *   B_{s,k}         byte for byte row list[k] of aclb200_decompress_bones with the same parents and ACLB200_OBJECT_QVVF for {clip, u'}.
 *   row             F = rtm::qvv_mul(rtm::qvv_mul(B, rtm::qvv_inverse(T_s)), M_s), both branches of qvv_mul: the bone at time t + offsets[s]
 *                   in the root's frame at time t. When the root track is a root of the skeleton, its own entry is M_s up to rounding (the
 *                   trajectory). Velocities are differences of two offsets' translations.
 *   d_out           row (s, k) of request r at d_out + r * pose_stride + (s * K + k) * 48, 48 byte rows of the ACLB200_OBJECT_QVVF layout, 16
 *                   byte aligned; pose_stride = options->pose_stride_bytes, 0 = S * K * 48.
 *   untouched       every row of a request with an invalid clip index, a list index >= num_lists, a root at or beyond its clip's num_tracks
 *                   or a looping value other than 0 and 1; the K rows of an offset whose u is not finite under ACLB200_FEATURE_LOOP or whose
 *                   |c| > ACLB200_MAX_ROOT_MOTION_CYCLES; the row of an entry that is ACLB200_NO_BONE or at or beyond its clip's num_tracks.
 *   d_out_flags     device uint32, optional: cleared, then OR-ed in: ACLB200_ERROR_FLAG_NEGATIVE_SCALE when a qvv_mul of the walk, of M or of
 *                   F took its matrix branch; ACLB200_ERROR_FLAG_INVALID_SKELETON from the walk; ACLB200_ERROR_FLAG_WRAP_CLIP_CYCLE when an
 *                   offset that writes its rows has c != 0 on a clip compressed with the wrap policy (as aclb200_extract_root_motion).
 * As aclb200_decompress_bones and aclb200_extract_root_motion: a bound database's streamed tiers are read, variable defaults and the batch
 * and per track rounding policies are honoured, ACLB200_MATH_FAST is accepted and runs the exact decode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing and leaving *d_out_flags untouched: NULL offsets, a non-finite offset,
 * num_offsets 0 or above ACLB200_MAX_FEATURE_OFFSETS, num_requests * num_offsets above 2^32 - 1, NULL d_parent_indices, the bone list
 * refusals of aclb200_decompress_bones, the refusals of aclb200_extract_root_motion (output_layout other than QVV48, looping_policy other
 * than ACLB200_LOOP_CLAMP, d_request_policies, skip masks or a `skipped` default mode, a scalar clip set), NULL d_requests or d_out with
 * num_requests > 0, a pose stride below S * K * 48, rows not 16 byte aligned. ACLB200_ERR_UNSUPPORTED when one pose of the widest clip does
 * not fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_extract_pose_features(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_feature_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const float* offsets, uint32_t num_offsets,
	const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list, const uint32_t* d_request_lists,
	const uint32_t* d_root_tracks, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* ---- Motion matching: pose feature rows packed into vectors, and the best database row of each query ---------------------------- */

/* aclb200_feature_term::kind */
#define ACLB200_FEATURE_POSITION 0u		/* the translation of row (s0, k) */
#define ACLB200_FEATURE_DIRECTION 1u	/* rtm::quat_mul_vector3(e_axis, rotation of row (s0, k)): where the bone's local axis points */
#define ACLB200_FEATURE_VELOCITY 2u		/* (translation of row (s1, k) - translation of row (s0, k)) * inv_dt */
/* The most dimensions of a packed feature vector */
#define ACLB200_MAX_FEATURE_DIMS 64
/* aclb200_search_result::row of a query without a candidate */
#define ACLB200_NO_ROW 0xFFFFFFFFu

/* One term of a feature vector: 1 to 3 of the x, y, z components of one vector taken from the rows of one request */
typedef struct aclb200_feature_term
{
	uint32_t kind;				/* ACLB200_FEATURE_* */
	uint32_t s0;				/* the offset of the row read (VELOCITY: the earlier one), 0..S-1 */
	uint32_t s1;				/* VELOCITY: the offset of the later row, 0..S-1; unused otherwise */
	uint32_t k;					/* the bone list entry, 0..K-1 */
	uint32_t axis;				/* DIRECTION: 0, 1 or 2 = the unit x, y or z axis; unused otherwise */
	uint32_t components;		/* bit mask of the components emitted, x = 1, y = 2, z = 4 (1..7), always in x, y, z order */
	float    inv_dt;			/* VELOCITY: 1 / the time between the two offsets; unused otherwise */
} aclb200_feature_term;

/* Pack pose features into vectors: request r's rows of aclb200_extract_pose_features (S = num_offsets, K = bones_per_list; row (s, k) at
 * d_rows + r * pose_stride + (s * K + k) * 48, pose_stride = pose_stride_bytes, 0 = S * K * 48, 16 byte aligned) become one vector of D =
 * num_dims floats at d_out + r * out_stride. The terms (a HOST array of num_terms, copied into the launch) emit their components in array
 * order, each term its components in x, y, z order; D must be the sum of their component counts.
 *   POSITION    v = t(s0, k)_c
 *   DIRECTION   v = rtm::quat_mul_vector3(e_axis, q(s0, k))_c, the rotation function of the object space walk
 *   VELOCITY    v = (t(s1, k)_c - t(s0, k)_c) * inv_dt, an IEEE subtract then multiply, not fused
 *   out[r][d]   (v_d - mean[d]) * scale[d], not fused; mean and scale are HOST float[D], NULL reads as 0 and 1 with the same arithmetic.
 * out_stride is in floats, at least D and a multiple of 4; d_out is 16 byte aligned; the floats from D to out_stride are not written. The
 * pack does not know which rows extract_pose_features left untouched: a caller tags such requests' database rows out of the search.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: an unknown kind, s0 or s1 >= S, k >= K, axis > 2, components 0 or above 7,
 * a non-finite inv_dt, mean or scale, num_terms 0 or NULL terms, D not the sum of the terms' components or above ACLB200_MAX_FEATURE_DIMS,
 * num_offsets 0 or above ACLB200_MAX_FEATURE_OFFSETS, bones_per_list 0 or above ACLB200_MAX_QUERY_BONES, a pose stride below S * K * 48 or
 * not a multiple of 16, NULL or misaligned d_rows or d_out with num_requests > 0. */
ACLB200_API aclb200_status aclb200_pack_pose_features(aclb200_context* context, const void* d_rows, uint32_t num_requests, uint32_t num_offsets,
	uint32_t bones_per_list, uint64_t pose_stride_bytes, const aclb200_feature_term* terms, uint32_t num_terms, const float* mean,
	const float* scale, uint32_t num_dims, float* d_out, uint32_t out_stride, void* stream);

/* What one query searches */
typedef struct aclb200_search_query
{
	uint32_t tag_mask;			/* row r is allowed when (d_row_tags[r] & tag_mask) != 0 */
	uint32_t exclude_begin;		/* rows exclude_begin <= r < exclude_end are skipped (the clip and time the character plays now); */
	uint32_t exclude_end;		/* begin >= end skips nothing */
} aclb200_search_query;

/* A query's best row. Read as a little endian uint64 it is (cost bits << 32) | row, the key the search minimises. */
typedef struct aclb200_search_result
{
	uint32_t row;				/* ACLB200_NO_ROW when the query has no candidate */
	float    cost;				/* +inf when the query has no candidate */
} aclb200_search_result;

/* The best database row of each query, exact and tie-stable, in one pass over the database. Database row r is D = num_dims floats at
 * d_database + r * db_stride (r < num_rows), query q's vector at d_query_vectors + q * q_stride.
 *   cost        acc = +0.0f; for d = 0 .. D-1 in order: diff = q[d] - x[d] (IEEE subtract); acc = fmaf(diff, diff, acc), a fused multiply add
 *               (correctly rounded, as C's fmaf). Never negative.
 *   candidate   row r with exclude_begin <= r < exclude_end false, (tag[r] & tag_mask) != 0 and a cost that is not NaN (+inf is a candidate);
 *               tag[r] = d_row_tags[r] (device uint32[num_rows]), every tag 0xFFFFFFFF when d_row_tags is NULL.
 *   result      d_results[q] (device, 8 byte aligned) = the candidate with the smallest cost, the lowest row among equal costs; {ACLB200_NO_ROW,
 *               +inf} without a candidate (every query when num_rows is 0).
 * The result does not depend on the launch shape or the order blocks run in: two launches give the same bits. d_queries is device
 * aclb200_search_query[num_queries].
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing and leaving d_results untouched: D 0 or above ACLB200_MAX_FEATURE_DIMS, a
 * stride below D or not a multiple of 4 floats, vectors not 16 byte aligned, results not 8 byte aligned, num_rows >= 2^32 - 1, NULL
 * d_database with num_rows > 0, NULL d_query_vectors, d_queries or d_results with num_queries > 0. */
ACLB200_API aclb200_status aclb200_search_pose_features(aclb200_context* context, const float* d_database, uint64_t num_rows, uint64_t db_stride,
	const uint32_t* d_row_tags, const float* d_query_vectors, const aclb200_search_query* d_queries, uint32_t num_queries, uint64_t q_stride,
	uint32_t num_dims, aclb200_search_result* d_results, void* stream);

/* Inertialization: hiding the jump when a character changes clips (a motion matching search result, a state change) without a crossfade.
 * At the jump, aclb200_begin_inertialization records per bone the offset from the pose the character displayed to the destination pose,
 * with the offset's velocity. From then on only the destination clip is decoded, and aclb200_inertialize_poses adds the offset as a
 * critically damped spring decays it to zero. Jumps chain: the next capture starts from the displayed pose, which holds the offset.
 *
 * Notation: quat_mul(a, b) is rtm's (apply a, then b: the Hamilton product b a); conj(q) negates x, y and z; abs(q) negates all four lanes
 * when q.w < 0.0f (an IEEE compare: -0 is kept); log and exp are rtm::quat_rotation_log and rtm::quat_rotation_exp (quatf.h:1306-1375) on
 * their SSE2 paths, with their near identity and near zero selects; the sin, cos and acos inside them are rtm's polynomials. Every
 * operation is IEEE and unfused: the results are those of the reference's rtm on any CPU, bit for bit.
 *
 * The record: per bone one 64 byte entry of four float4, each xyz plus w = 0; a record is num_tracks entries, 16 byte aligned, in device
 * memory the caller owns. A caller may write entries directly: for example zeroing the root bone's entry when the root moves by
 * aclb200_extract_root_motion.
 *   rot_x  rotation offset as a scaled angle axis: 2 log(abs(quat_mul(conj(dst.q), src.q))).xyz (the Hamilton src dst^-1)
 *   rot_v  angular velocity offset: w(src) - w(dst), w(p) = (2 log(abs(quat_mul(conj(p_prev.q), p.q))).xyz) * inv_dt
 *   pos_x  translation offset: src.t - dst.t
 *   pos_v  linear velocity offset: v(src) - v(dst), v(p) = (p.t - p_prev.t) * inv_dt
 * Scale is not inertialized (the output takes the destination's scale), so an entry is 64 bytes rather than 96. */
#define ACLB200_NO_INERTIALIZATION 0xFFFFFFFFu
#define ACLB200_INERTIALIZATION_ENTRY_BYTES 64u

/* One pose's decay: the record it reads (ACLB200_NO_INERTIALIZATION: none), the seconds since its capture and the spring's halflife in
 * seconds, both used as given (no clamp). 12 bytes, 4 byte aligned. */
typedef struct aclb200_inertialization
{
	uint32_t record;
	float    elapsed;
	float    halflife;
} aclb200_inertialization;

/* The capture: transition j reads four QVV48 local poses of one skeleton (rtm::qvvf rows, 48 byte bones, 16 byte aligned, pose j of each
 * buffer at j * pose_stride_bytes, 0 = num_tracks * 48): the displayed pose this frame (d_src) and the frame before (d_src_prev), and the
 * destination pose this frame (d_dst) and the frame before (d_dst_prev), one frame being 1 / inv_dt seconds. It writes the num_tracks
 * entries of the record at d_records + slot * record_stride_bytes (0 = num_tracks * 64), slot = d_record_slots[j] (device
 * uint32[num_transitions]) or j when d_record_slots is NULL. Slots are the caller's to keep in range and distinct.
 * The displayed poses are what the character showed: its current clip decoded at both times with aclb200_inertialize_poses applied with
 * its current record (or none). The destination poses come from one aclb200_decompress_tracks launch with two requests per transition.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: NULL or misaligned poses or records with num_transitions > 0, a record
 * stride below num_tracks * 64 or not a multiple of 16, a slot list not 4 byte aligned, an inv_dt that is zero or not finite. */
ACLB200_API aclb200_status aclb200_begin_inertialization(aclb200_context* context, const void* d_src, const void* d_src_prev, const void* d_dst,
	const void* d_dst_prev, uint64_t num_transitions, uint32_t num_tracks, uint64_t pose_stride_bytes, float inv_dt, void* d_records,
	uint64_t record_stride_bytes, const uint32_t* d_record_slots, void* stream);

/* The apply, on num_poses QVV48 poses already on the device (a decode, a blend, a layer stack; pose p at p * pose_stride_bytes in d_poses
 * and d_out, 0 = num_tracks * 48). Pose p takes d_inertializations[p] (device) and, unless its record is ACLB200_NO_INERTIALIZATION, the
 * record at d_records + record * record_stride_bytes (0 = num_tracks * 64). Per pose, from its elapsed and halflife:
 *     y = (2.7725887f / (halflife + 1e-5f)) * 0.5f;   u = y * elapsed
 *     e = 1.0f / (((1.0f + u) + (0.48f * u) * u) + ((0.235f * u) * u) * u)
 *     x(x0, v0) = e * (x0 + (v0 + x0 * y) * elapsed)          per component, in this order
 * and per bone: rotation quat_mul(dst.q, exp(x(rot_x, rot_v) * 0.5f)) (the Hamilton offset dst), translation dst.t + x(pos_x, pos_v),
 * scale dst.s; the translation and scale w lanes are written as 0. Nothing is normalised beyond what rtm's functions do.
 * A pose whose record is ACLB200_NO_INERTIALIZATION is copied unchanged; a pose whose record is >= num_records is not written. d_out may
 * be d_poses. A record with fewer entries than num_tracks is the caller's error, as for skeleton offsets.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: NULL or misaligned poses, NULL or misaligned (4 byte) d_inertializations
 * with num_poses > 0, NULL or misaligned (16 byte) d_records with num_records > 0, a record stride below num_tracks * 64 or not a
 * multiple of 16, num_records >= 2^32 - 1. */
ACLB200_API aclb200_status aclb200_inertialize_poses(aclb200_context* context, const void* d_poses, void* d_out, uint64_t num_poses,
	uint32_t num_tracks, uint64_t pose_stride_bytes, const aclb200_inertialization* d_inertializations, const void* d_records,
	uint64_t num_records, uint64_t record_stride_bytes, void* stream);

/* One request of the inertialized decode: the pose to decode and its inertialization. 20 bytes, 4 byte aligned. */
typedef struct aclb200_inertialized_request
{
	aclb200_request         pose;
	aclb200_inertialization inertialization;
} aclb200_inertialized_request;

/* The decode and the apply in one launch, the per-frame call of characters in transition: request r is decoded as aclb200_decompress_tracks
 * decodes its pose, then, before the rows leave shared memory, the record's offset is decayed onto them exactly as aclb200_inertialize_poses
 * computes it (QVV48 and QVV40 rows). With parents (d_parent_indices, d_skeleton_offsets and object_kind as aclb200_decompress_tracks_blend)
 * the inertialized local pose is then taken to object space, as qvvf or 3x4 matrix rows; without them the rows stay local, in
 * options->output_layout. Records at d_records + record * record_stride_bytes (0 = max_tracks * 64), 16 byte aligned.
 *   record == ACLB200_NO_INERTIALIZATION   the request reads no record: its rows are byte for byte those of aclb200_decompress_tracks (no
 *                                          parents), aclb200_decompress_tracks_object_space or _skinning for the same request and options,
 *                                          so characters not in transition share the launch at no extra traffic
 *   record >= num_records, invalid clip     nothing is written for the request
 * A record with fewer entries than the clip's tracks is the caller's error, as for skeleton offsets. d_out_flags as the object space
 * decode; the inertialization raises no flags. ACLB200_MATH_FAST is accepted and runs the exact decode, as in every composed mode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: the refusals of aclb200_decompress_tracks_blend (skip masks, a `skipped`
 * default mode, a scalar clip set, alignment, an unknown object_kind, QVV40 with parents), a record stride below max_tracks * 64 or not a
 * multiple of 16, NULL or misaligned d_records with num_records > 0, num_records >= 2^32 - 1, NULL requests or output with a count above 0.
 * ACLB200_ERR_UNSUPPORTED when one pose does not fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_inertialized(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_inertialized_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const void* d_records, uint64_t num_records, uint64_t record_stride_bytes,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The skinning rows of the inertialized pose: aclb200_decompress_tracks_inertialized through the matrix walk and the skinning step of
 * aclb200_decompress_tracks_skinning (parents and inverse binds required). */
ACLB200_API aclb200_status aclb200_decompress_tracks_inertialized_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_inertialized_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const void* d_records, uint64_t num_records, uint64_t record_stride_bytes,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* Mirroring: playing a clip left/right mirrored, so that a motion matching database holds each clip twice (as recorded and mirrored)
 * while only the recorded copy is authored and compressed. Each row of the mirrored pose takes the transform of its mirror row (left
 * hand from right hand), reflected across a plane through the origin and corrected for the difference between the two bones' frames.
 *
 * Notation as for inertialization: quat_mul(a, b) is rtm's (apply a, then b: the Hamilton product b a), quat_mul_vector3(v, q) is rtm's
 * (v rotated by q). Every operation is IEEE and unfused; the results equal the reference's rtm::quat_mul and quat_mul_vector3 on any CPU.
 *
 * The mirror axis, the normal of the mirror plane: ACLB200_MIRROR_X, _Y or _Z.
 *   reflect_q(q)   flips the sign bits of the two quaternion vector lanes other than `axis` (X: (x, -y, -z, w))
 *   reflect_t(t)   flips the sign bit of lane `axis` of the translation (X: (-x, y, z))
 * Both are sign flips, not subtractions: +0 and -0 swap and NaN payloads are kept.
 *
 * The mirror table: one aclb200_mirror_entry per row, 16 byte aligned, in device memory the caller owns. Row i of a pose of n rows has
 * the partner m = entry[i].mirror when m < n and entry[m].mirror == i; otherwise its partner is i itself and
 * ACLB200_ERROR_FLAG_INVALID_MIRROR is raised. Partners therefore always pair up. For row i with partner m:
 *   rotation      quat_mul(quat_mul(entry[i].pre, reflect_q(q_m)), entry[i].post)
 *   translation   quat_mul_vector3(reflect_t(t_m), entry[i].post)
 *   scale         s_m, the bits copied
 * The w lanes of translation and scale are written as 0 (QVV48). Nothing is normalised, and the quat_muls run for identity corrections too.
 *
 * In matrix terms the row is C_frame^-1 S X_m S C_i, with S the reflection, pre = C_i and post = conj(C_frame): C_i is the correction
 * that takes row i's reflected frame to its own, and the frame is what the row is relative to. One table format serves every kind of row:
 *   local pose rows     frame = the bone's parent (identity for roots); api.py's mirror_table builds this table from a bind pose
 *   object rows         frame = identity (post = identity)
 *   feature rows        (aclb200_extract_pose_features, relative to the root) frame = the root
 *   root motion rows    pre = C_root, post = conj(C_root)
 * Scale is copied, which is exact when each correction maps every axis onto plus or minus itself (identity, or a half turn about x, y or
 * z): the corrections rigs use. Corrections that swap axes under non-uniform scale are the caller's responsibility. */
#define ACLB200_MIRROR_X 0u
#define ACLB200_MIRROR_Y 1u
#define ACLB200_MIRROR_Z 2u

/* One row's mirror table entry: 48 bytes, 16 byte aligned. */
typedef struct aclb200_mirror_entry
{
	float    pre[4];		/* quaternion xyzw applied before the reflected rotation */
	float    post[4];		/* quaternion xyzw applied after it, and to the translation */
	uint32_t mirror;		/* the row this row takes its transform from */
	uint32_t reserved[3];	/* ignored */
} aclb200_mirror_entry;

/* Mirrors num_poses poses of QVV48 rows already on the device: decodes, blends, layer stacks, pose feature rows (num_rows = K, one pose
 * per (request, offset)), root motion rows (num_rows = 1). Pose p has num_rows rows at p * pose_stride_bytes in d_poses and d_out
 * (0 = num_rows * 48); row i takes the table entry d_table[i]. d_mirrored (device uint32[num_poses], optional) says per pose:
 *   NULL   every pose is mirrored
 *   0      the pose is copied unchanged
 *   1      the pose is mirrored
 *   other  the pose is not written
 * d_out may be d_poses. d_out_flags: device uint32, optional: cleared, then ACLB200_ERROR_FLAG_INVALID_MIRROR OR-ed in when a mirrored
 * pose met an entry without a partner.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: an unknown axis; NULL or misaligned (16 byte) poses or table, or a
 * misaligned (4 byte) d_mirrored, with num_poses and num_rows above 0; a pose stride below num_rows * 48 or not a multiple of 16. */
ACLB200_API aclb200_status aclb200_mirror_poses(aclb200_context* context, const void* d_poses, void* d_out, uint64_t num_poses, uint32_t num_rows,
	uint64_t pose_stride_bytes, const uint32_t* d_mirrored, const aclb200_mirror_entry* d_table, uint32_t axis, uint32_t* d_out_flags,
	void* stream);

/* One request of the mirrored decode: the pose to decode and whether to mirror it. 12 bytes, 4 byte aligned. */
typedef struct aclb200_mirrored_request
{
	aclb200_request pose;
	uint32_t        mirrored;
} aclb200_mirrored_request;

/* The decode and the mirror in one launch: request r is decoded as aclb200_decompress_tracks decodes its pose; when mirrored == 1 the
 * rows are then mirrored in shared memory exactly as aclb200_mirror_poses mirrors them (QVV48 and QVV40 rows). Clip c's table starts at
 * d_mirror_table + d_skeleton_offsets[c] (0 when d_skeleton_offsets is NULL): it is indexed like the parents, so a mirror table belongs to
 * a skeleton. With parents (d_parent_indices, d_skeleton_offsets and object_kind as aclb200_decompress_tracks_blend) the pose is then
 * taken to object space, as qvvf or 3x4 matrix rows, by the walk of aclb200_local_to_object_space; without them the rows stay local, in
 * options->output_layout.
 *   mirrored == 0                          the rows are byte for byte those of aclb200_decompress_tracks (no parents),
 *                                          aclb200_decompress_tracks_object_space or _skinning for the same request and options
 *   mirrored == 1                          the rows are byte for byte aclb200_mirror_poses of the decoded local pose, then the walk and
 *                                          skinning of aclb200_local_to_object_space or aclb200_local_to_skinning
 *   any other value, invalid clip          nothing is written for the request, and it is not sought
 * d_out_flags as the object space decode, plus ACLB200_ERROR_FLAG_INVALID_MIRROR. ACLB200_MATH_FAST is accepted and runs the exact
 * decode, as in every composed mode.
 * Refused with ACLB200_ERR_INVALID_ARGUMENT, launching nothing: the refusals of aclb200_decompress_tracks_inertialized (skip masks, a
 * `skipped` default mode, a scalar clip set, alignment, an unknown object_kind, QVV40 with parents, NULL requests or output with a count
 * above 0), an unknown axis, a NULL or misaligned (16 byte) table with num_requests > 0. ACLB200_ERR_UNSUPPORTED when one pose does not fit
 * in a block's shared memory. */
ACLB200_API aclb200_status aclb200_decompress_tracks_mirrored(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const aclb200_mirror_entry* d_mirror_table, uint32_t axis,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The skinning rows of the mirrored pose: aclb200_decompress_tracks_mirrored through the matrix walk and the skinning step of
 * aclb200_decompress_tracks_skinning (parents and inverse binds required). */
ACLB200_API aclb200_status aclb200_decompress_tracks_mirrored_skinning(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options* options,
	const aclb200_mirror_entry* d_mirror_table, uint32_t axis,
	const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
	void* d_out, uint32_t* d_out_flags, void* stream);

/* The skinning rows of aclb200_decompress_tracks_skinning for poses already on the device (the end of an aclb200_blend_poses chain, of
 * aclb200_apply_additive_to_base): num_poses poses of rtm::qvvf rows of one skeleton (48 byte bones, 16 byte aligned, pose p at
 * p * pose_stride_bytes in both buffers, 0 = num_tracks * 48) in, skinning rows out, bit-identical to the fused route. The skeleton is
 * d_parent_indices and the inverse binds d_inverse_bind, both at offset 0. d_out may be d_local_poses. d_out_flags as
 * aclb200_local_to_object_space. Refused with ACLB200_ERR_INVALID_ARGUMENT: NULL pointers, misaligned rows or inverse binds;
 * ACLB200_ERR_UNSUPPORTED when one pose does not fit in a block's shared memory. */
ACLB200_API aclb200_status aclb200_local_to_skinning(aclb200_context* context, const void* d_local_poses, void* d_out, uint64_t num_poses,
	uint32_t num_tracks, uint64_t pose_stride_bytes, const uint32_t* d_parent_indices, const float* d_inverse_bind, uint32_t* d_out_flags,
	void* stream);

/* Parity / debugging hooks (integer stages of the decode, bit-exact against the reference):
 *  - aclb200_debug_seek: the state seek_v0 computes, one aclb200_seek_state per request (device output).
 *  - aclb200_debug_unpack: for request r and key frame `which` (0/1), writes one uint4 per animated sub-track
 *    (rotations, translations, scales order): x, y, z quantised integers (or raw float bits) and the stored
 *    per-track bit count, at d_out + r * max_animated_sub_tracks * 16 bytes.
 * Both return ACLB200_ERR_UNSUPPORTED on a clip set whose bound database has chunks streamed in. */
ACLB200_API aclb200_status aclb200_debug_seek(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, aclb200_seek_state* d_out, void* stream);
ACLB200_API aclb200_status aclb200_debug_unpack(aclb200_context* context, const aclb200_clipset* clipset,
	const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, uint32_t which,
	uint32_t max_animated_sub_tracks, uint32_t* d_out, void* stream);

/* Profiling hook of the pipeline kernel (only builds compiled with -DACLB200_PIPE_TRACE=1 write anything): the first
 * `num_blocks` blocks record 8 clock64() stamps per batch they decode, for their first `num_iterations` batches, at
 * d_trace[(block * num_iterations + iteration) * 8 + k] (uint64). NULL switches it off. tools/pipe_trace.py reads it. */
ACLB200_API aclb200_status aclb200_debug_set_trace(aclb200_context* context, void* d_trace, uint32_t num_blocks, uint32_t num_iterations);

/* Which kernel the latest aclb200_decompress_tracks on a context launched, and the plan of that launch. Tests use it to check that
 * a request list really reaches the pipeline configuration it was written for (several batches per block, one request per batch,
 * the plain kernels when a pose does not fit in shared memory). */
enum { ACLB200_KERNEL_NONE = 0, ACLB200_KERNEL_PLAIN = 1, ACLB200_KERNEL_PIPELINE = 2, ACLB200_KERNEL_DATABASE = 3 };

typedef struct aclb200_launch_info
{
	uint32_t kernel;				/* ACLB200_KERNEL_*: NONE before the first launch with at least one request */
	uint32_t requests_per_block;	/* requests per batch (pipeline) or per block (plain and database kernels) */
	uint32_t grid_blocks;			/* blocks launched: the pipeline's persistent grid walks num_batches / grid_blocks batches per block */
	uint32_t num_batches;			/* ceil(num_requests / requests_per_block) */
	uint32_t out_bulk;				/* pipeline: 1 when pose rows leave shared memory as TMA bulk stores, 0 for 8 byte stores; 0 otherwise */
	uint32_t num_requests;
} aclb200_launch_info;

ACLB200_API aclb200_status aclb200_debug_last_launch(const aclb200_context* context, aclb200_launch_info* out_info);

/* Plain device memory helpers so that a host language without the CUDA runtime can hand device arrays (requests, variable
 * defaults, per track policies, skip masks, outputs) to the entry points above. Synchronous. */
ACLB200_API aclb200_status aclb200_device_malloc(aclb200_context* context, size_t bytes, void** out_device_pointer);
ACLB200_API void aclb200_device_free(aclb200_context* context, void* device_pointer);
ACLB200_API aclb200_status aclb200_copy_to_device(aclb200_context* context, void* device_destination, const void* host_source, size_t bytes);
ACLB200_API aclb200_status aclb200_copy_to_host(aclb200_context* context, void* host_destination, const void* device_source, size_t bytes);

/* Number of kernels launched by this context so far (bench.py reports it as `gpu_launches`). */
ACLB200_API uint64_t aclb200_launch_count(const aclb200_context* context);

#ifdef __cplusplus
}
#endif

#endif /* ACLB200_H */
