// acl_b200/csrc/api.cpp -- the extern "C" surface declared in include/aclb200.h.
#include "context.h"

#include <cmath>
#include <cstddef>
#include <cstring>
#include <functional>
#include <new>

namespace aclb200
{
	aclb200_status build_clipset(aclb200_context* context, const std::function<const uint8_t*(uint32_t)>& get_blob, const uint32_t* sizes,
		uint32_t num_clips, bool check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip);

	namespace
	{
		uint32_t scalar_components(uint32_t track_type)
		{
			return track_type <= 3 ? track_type + 1 : 4;
		}

		// `skipped` default sub-tracks and skipped sub-tracks (track_writer::skip_*) keep what the caller's buffer holds
		bool keeps_caller_bytes(const aclb200_options& options)
		{
			return options.default_rotation_mode == ACLB200_DEFAULT_SKIPPED || options.default_translation_mode == ACLB200_DEFAULT_SKIPPED
				|| options.default_scale_mode == ACLB200_DEFAULT_SKIPPED || (options.skip_mask & 7u) != 0 || options.d_skip_track_mask != nullptr;
		}

		// What a composed entry point launches: pose r is the launch's requests r L .. r L + L - 1, combined by the compose mode
		struct Composed
		{
			const char* entry;						// the C entry point, for messages
			const char* unfit;						// the refusal of a pose whose requests do not fit one block's shared memory
			uint32_t compose;						// k_compose_*
			uint32_t num_layers;					// L: 1 (object), 2 (additive, blend) or the layered decode's num_layers
			float weight;							// blend: the weight of every pair when d_weights is NULL
			const float* d_weights;					// blend: [pairs] the weight of each pair, or NULL
			uint32_t additive_format;				// additive, layers: the format when d_clip_additive_formats is NULL
			const uint8_t* d_clip_additive_formats;	// additive, layers: [num_clips] the format of each clip, or NULL
			// layers_masked: the mask table (every field 0 in the other modes)
			const uint32_t* d_layer_masks;			// [num_poses * num_layers] the mask index of each layer, or NULL
			const float* d_bone_masks;				// [num_masks][mask_stride]
			uint32_t num_masks;
			uint32_t mask_stride;					// resolved by check_layer_masks (0 = max_tracks)
			// inertialize: the records (every field 0 in the other modes)
			const void* d_records;
			uint64_t record_stride;					// resolved by check_records (0 = max_tracks * 64)
			uint64_t num_records;
			// mirror: the table of skeleton 0 and the axis (every field 0 in the other modes)
			const aclb200_mirror_entry* d_mirror_table;
			uint32_t mirror_axis;
		};
		const char* const k_pose_unfit = ": one pose does not fit in a block's shared memory";
		const char* const k_pair_unfit = ": the two poses of a pair do not fit in a block's shared memory";
		const char* const k_layers_unfit = ": the poses of a layer stack do not fit in a block's shared memory";

		// what every decode checks before it reads an option: the handles, and an options struct of this library's size
		aclb200_status check_handles_and_options(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_options* options)
		{
			if (context == nullptr || clipset == nullptr || options == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
			if (options->struct_size != sizeof(aclb200_options))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "options.struct_size does not match this library, call aclb200_default_options()");
			return ACLB200_OK;
		}

		// The checks every decode shares and the DecodeParams they describe; a launch's own fields (its plan, its operands) are left 0
		aclb200_status make_params(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_request* d_requests,
			uint32_t num_requests, const aclb200_options* options, void* d_out, bool want_transform, bool single_track, DecodeParams& params)
		{
			const aclb200_status checked = check_handles_and_options(context, clipset, options);
			if (checked != ACLB200_OK)
				return checked;
			if (num_requests != 0 && (d_requests == nullptr || d_out == nullptr))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null request / output pointer");
			if (clipset->device != context->device)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "clip set lives on another device");
			const bool is_transform = clipset->info.track_type == ACLB200_TRACK_QVVF;
			if (is_transform != want_transform)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, want_transform ? "not a transform clip set" : "not a scalar clip set");
			if (options->rounding_policy > ACLB200_ROUND_PER_TRACK || options->looping_policy > ACLB200_LOOP_AS_COMPRESSED
				|| options->normalization > ACLB200_NORMALIZE_ALWAYS || options->output_layout > ACLB200_LAYOUT_QVV40
				|| options->default_rotation_mode > ACLB200_DEFAULT_VARIABLE || options->default_translation_mode > ACLB200_DEFAULT_VARIABLE
				|| options->default_scale_mode > ACLB200_DEFAULT_LEGACY)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "option value out of range");
			// ACL_ASSERT(rounding_policy != per_track || is_per_track_rounding_supported()), decompress.impl.h:211
			if (options->rounding_policy == ACLB200_ROUND_PER_TRACK && !options->per_track_rounding)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "per track rounding must be enabled to seek with the per_track policy");

			// the per track rounding kernels read one batch wide seek policy for the tracks that do not override it
			if (options->d_request_policies != nullptr && options->per_track_rounding)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "per request policies (d_request_policies) need per_track_rounding == 0");

			std::memset(&params, 0, sizeof(params));
			params.data = clipset->d_data;
			params.clips = clipset->d_clips;
			params.requests = d_requests;
			params.num_requests = num_requests;
			params.num_clips = clipset->info.num_clips;
			params.max_tracks = clipset->info.max_tracks;
			for (int k = 0; k < 3; ++k)
				params.max_animated[k] = clipset->max_animated[k];
			params.out = static_cast<uint8_t*>(d_out);
			if (is_transform)
				params.bone_stride = options->output_layout == ACLB200_LAYOUT_QVV48 ? 48u : 40u;
			else
				params.bone_stride = scalar_components(clipset->info.track_type) * 4u;
			params.pose_stride = options->pose_stride_bytes != 0 ? options->pose_stride_bytes : uint64_t(params.max_tracks) * params.bone_stride;
			if (!single_track && params.pose_stride < uint64_t(params.max_tracks) * params.bone_stride)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "pose_stride_bytes is smaller than one pose");
			if (is_transform)
			{
				const uint64_t alignment = options->output_layout == ACLB200_LAYOUT_QVV48 ? 16 : 8;
				if ((params.pose_stride % alignment) != 0 || (reinterpret_cast<uintptr_t>(d_out) % alignment) != 0)
					return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "the output pointer and pose_stride_bytes must keep bones 16 (QVV48) / 8 (QVV40) byte aligned");
			}
			else
			{
				// the scalar kernels store each component with one 4 byte store: a misaligned row would fault on the device
				const uint64_t misaligned = reinterpret_cast<uintptr_t>(d_out) | (single_track ? 0u : params.pose_stride);
				if ((misaligned % 4) != 0)
					return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, single_track ? "the output pointer must be 4 byte aligned"
						: "the output pointer and pose_stride_bytes must be multiples of 4");
			}
			params.rounding_policy = options->rounding_policy;
			params.looping_policy = options->looping_policy;
			params.normalization = options->normalization;
			params.per_track_rounding = options->per_track_rounding != 0;
			params.wrapping = options->wrapping != 0;
			params.clamp_sample_time = options->clamp_sample_time != 0;
			params.multiple_rotation_formats = options->multiple_rotation_formats != 0;
			params.default_mode[0] = options->default_rotation_mode;
			params.default_mode[1] = options->default_translation_mode;
			params.default_mode[2] = options->default_scale_mode;
			std::memcpy(params.constant_defaults, options->constant_defaults, sizeof(params.constant_defaults));
			params.variable_defaults = options->d_variable_defaults;
			params.per_track_policies = options->d_per_track_rounding;
			params.skip_all = is_transform ? (options->skip_mask & 7u) : 0u;
			params.skip_tracks = is_transform ? options->d_skip_track_mask : nullptr;
			params.request_policies = options->d_request_policies;
			params.layout = options->output_layout;
			// a bound database with chunks streamed in: the launch takes the database kernels (with nothing streamed in, the resident key
			// frames give the reference's result, so every other launch runs the kernels it always did)
			if (is_transform && database_streamed_in(clipset))
			{
				params.db_first_segment = clipset->d_db_first_segment;
				params.db_tiers = clipset->database->d_tiers;
				params.db_bulk[0] = clipset->database->d_bulk[0];
				params.db_bulk[1] = clipset->database->d_bulk[1];
			}
			params.num_layers = 1;
			return ACLB200_OK;
		}

		// an object transform needs every sub-track of its parents, apply_additive_to_base and qvv_lerp every sub-track of both poses:
		// the composed decodes, the bone query and root motion refuse skip masks and `skipped` default modes
		aclb200_status check_every_sub_track(aclb200_context* context, const aclb200_options& options, const std::string& entry)
		{
			if (keeps_caller_bytes(options))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry
					+ ": the composed poses need every decoded sub-track (no skip masks, no `skipped` default mode)");
			return ACLB200_OK;
		}

		// object space output (parents given): a known object kind, and QVV48 rows for the walk
		aclb200_status check_object_output(aclb200_context* context, const aclb200_options& options, const uint32_t* d_parent_indices,
			uint32_t object_kind, const std::string& entry)
		{
			if (d_parent_indices != nullptr && object_kind != ACLB200_OBJECT_QVVF && object_kind != ACLB200_OBJECT_MATRIX3X4F)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": unknown object_kind");
			if (d_parent_indices != nullptr && options.output_layout != ACLB200_LAYOUT_QVV48)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": object space output needs the QVV48 layout");
			return ACLB200_OK;
		}

		// the bone lists of the bone query and the pose features: K = bones_per_list of 1..32 entries, at least one list
		aclb200_status check_bone_lists(aclb200_context* context, const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list,
			const std::string& entry)
		{
			if (bones_per_list == 0 || bones_per_list > ACLB200_MAX_QUERY_BONES)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": bones_per_list must be 1 to 32");
			if (num_lists == 0 || d_bone_lists == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": needs at least one bone list (num_lists >= 1, d_bone_lists not NULL)");
			return ACLB200_OK;
		}

		// the root samples of root motion and the pose features: QVV48 rows, every one taken with the clamp looping policy
		aclb200_status check_root_samples(aclb200_context* context, const aclb200_options& options, const std::string& entry)
		{
			if (options.output_layout != ACLB200_LAYOUT_QVV48)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": the root samples and the output are QVV48 rows");
			if (options.looping_policy != ACLB200_LOOP_CLAMP)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": every root sample is taken with the clamp looping policy");
			if (options.d_request_policies != nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": per request policies would override the clamp looping policy");
			return ACLB200_OK;
		}

		aclb200_status finish_launch(aclb200_context* context, cudaError_t error, const char* what)
		{
			if (error == cudaSuccess)
				context->launch_count++;
			return check_cuda(context, error, what);
		}

		// The tail of a launch that ORs ACLB200_ERROR_FLAG_* into d_out_flags: on the context's device, the flags word is cleared on the
		// stream (a failure there is reported as `what`'s), then launch() runs and is counted when it started (reported as `route`'s)
		template<class Launch>
		aclb200_status launch_clearing_flags(aclb200_context* context, uint32_t* d_out_flags, cudaStream_t stream, const char* what, const char* route,
			Launch launch)
		{
			cudaSetDevice(context->device);
			const aclb200_status cleared = clear_out_flags(context, d_out_flags, stream, what);
			if (cleared != ACLB200_OK)
				return cleared;
			return finish_launch(context, launch(), route);
		}
	}

	aclb200_status clear_out_flags(aclb200_context* context, uint32_t* d_out_flags, cudaStream_t stream, const char* what)
	{
		return d_out_flags != nullptr ? check_cuda(context, cudaMemsetAsync(d_out_flags, 0, sizeof(uint32_t), stream), what) : ACLB200_OK;
	}

	aclb200_status check_qvvf_rows(aclb200_context* context, std::initializer_list<const void*> poses, uint32_t num_tracks, uint64_t& pose_stride,
		const char* what)
	{
		if (pose_stride == 0)
			pose_stride = uint64_t(num_tracks) * 48;
		uintptr_t addresses = 0;
		for (const void* pose : poses)
			addresses |= reinterpret_cast<uintptr_t>(pose);
		if (pose_stride < uint64_t(num_tracks) * 48 || (pose_stride % 16) != 0 || (addresses % 16) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": poses are rtm::qvvf rows (48 byte bones), 16 byte aligned");
		return ACLB200_OK;
	}

	// inertialization records: 64 byte entries per bone, 16 byte aligned; record_stride 0 becomes num_tracks * 64
	aclb200_status check_records(aclb200_context* context, const void* d_records, uint32_t num_tracks, uint64_t& record_stride, const char* what)
	{
		if (record_stride == 0)
			record_stride = uint64_t(num_tracks) * ACLB200_INERTIALIZATION_ENTRY_BYTES;
		if (record_stride < uint64_t(num_tracks) * ACLB200_INERTIALIZATION_ENTRY_BYTES || (record_stride % 16) != 0
			|| (reinterpret_cast<uintptr_t>(d_records) % 16) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": records are 64 byte entries per bone, 16 byte aligned");
		return ACLB200_OK;
	}

	// mirroring: a known axis, and a 16 byte aligned table wherever there is work to do
	aclb200_status check_mirror(aclb200_context* context, const aclb200_mirror_entry* d_table, uint32_t axis, bool work, const char* what)
	{
		if (axis > ACLB200_MIRROR_Z)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": axis must be ACLB200_MIRROR_X, _Y or _Z");
		if (work && (d_table == nullptr || (reinterpret_cast<uintptr_t>(d_table) % 16) != 0))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": the mirror table is 48 byte entries, 16 byte aligned, never NULL");
		return ACLB200_OK;
	}

	aclb200_status check_inverse_binds(aclb200_context* context, const float* d_inverse_bind, const char* what)
	{
		if (d_inverse_bind == nullptr || (reinterpret_cast<uintptr_t>(d_inverse_bind) % 16) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": inverse binds are 12 float matrices, 16 byte aligned, never NULL");
		return ACLB200_OK;
	}

	namespace
	{
		// what the two layered decodes check of their own: the stack depth, the launch's request count and the additive format
		aclb200_status check_layers(aclb200_context* context, uint32_t num_poses, uint32_t num_layers, uint32_t additive_format, const char* what)
		{
			if (num_layers == 0 || num_layers > k_max_layers)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": num_layers must be 1 to 8");
			if (uint64_t(num_poses) * num_layers > 0xFFFFFFFFu)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": num_poses * num_layers is above 2^32 - 1");
			if (additive_format > ACLB200_ADDITIVE_ADDITIVE1)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": additive_format out of range");
			return ACLB200_OK;
		}

		// what the two masked layered decodes check of their own: the mask table, when a layer may name a mask; fills the Composed's mask
		// fields (mask_stride 0 becomes max_tracks). A null clip set is left to make_params.
		aclb200_status check_layer_masks(aclb200_context* context, const aclb200_clipset* clipset, const uint32_t* d_layer_masks,
			const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const char* what, Composed& composed)
		{
			if (d_layer_masks == nullptr)
				return ACLB200_OK;
			if (d_bone_masks == nullptr || num_masks == 0)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": layer masks need d_bone_masks and num_masks >= 1");
			if ((reinterpret_cast<uintptr_t>(d_bone_masks) % 4) != 0)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": d_bone_masks must be 4 byte aligned");
			if (num_masks > k_max_layer_masks)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": num_masks is above 2^29 - 1");
			const uint32_t max_tracks = clipset != nullptr ? clipset->info.max_tracks : 0u;
			if (mask_stride == 0)
				mask_stride = max_tracks;
			if (mask_stride < max_tracks)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": mask_stride is below the clip set's max_tracks");
			if (uint64_t(num_masks) * mask_stride > 0xFFFFFFFFu)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": num_masks * mask_stride is above 2^32 - 1");
			composed.d_layer_masks = d_layer_masks;
			composed.d_bone_masks = d_bone_masks;
			composed.num_masks = num_masks;
			composed.mask_stride = mask_stride;
			return ACLB200_OK;
		}

		// The composed decodes: num_poses poses of composed.num_layers requests each at d_requests. Every refusal comes before the flags are
		// cleared: a refused call writes nothing. skinning (the _skinning entry points, which pass the matrix object kind): parents and
		// inverse binds are required, the walk's matrices are skinned (the object kind k_object_skinning).
		aclb200_status decompress_composed(aclb200_context* context, const aclb200_clipset* clipset, const void* d_requests, uint32_t num_poses,
			const aclb200_options* options, const Composed& composed, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
			uint32_t object_kind, bool skinning, const float* d_inverse_bind, void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const std::string entry = composed.entry;
			// the object space and skinning decodes require parents (the other modes take them to mean object space output), the skinning
			// decodes inverse binds too
			if (d_parent_indices == nullptr && (skinning || composed.compose == k_compose_object))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, entry + ": null parent index pointer");
			DecodeParams params;
			aclb200_status status = skinning ? check_inverse_binds(context, d_inverse_bind, composed.entry) : ACLB200_OK;
			if (status == ACLB200_OK)
				status = make_params(context, clipset, static_cast<const aclb200_request*>(d_requests), num_poses * composed.num_layers, options, d_out,
					true, false, params);
			if (status == ACLB200_OK)
				status = check_every_sub_track(context, *options, entry);
			// object space output: always in the object space decode (its entry point requires parents), with parents in the others
			if (status == ACLB200_OK)
				status = check_object_output(context, *options, d_parent_indices, object_kind, entry);
			if (status != ACLB200_OK)
				return status;
			// the poses stay in shared memory and give up key frame staging first: what is left must fit one block
			params.num_layers = composed.num_layers;
			plan_launch(params, clipset->max_key_frame_bytes, context->max_dynamic_smem, true, params.db_tiers != nullptr, composed.compose);
			if (params.smem_bytes > uint32_t(context->max_dynamic_smem > 0 ? context->max_dynamic_smem : 0))
				return set_error(context, ACLB200_ERR_UNSUPPORTED, entry + composed.unfit);
			if (num_poses == 0)
				return ACLB200_OK;
			params.parent_indices = d_parent_indices;
			params.skeleton_offsets = d_skeleton_offsets;
			params.object_flags = d_out_flags;
			params.object_kind = skinning ? k_object_skinning : object_kind;
			params.inverse_bind = d_inverse_bind;
			params.blend_weight = composed.weight;
			params.blend_weights = composed.d_weights;
			params.additive_format = composed.additive_format;
			params.clip_additive_formats = composed.d_clip_additive_formats;
			params.layer_masks = composed.d_layer_masks;
			params.bone_masks = composed.d_bone_masks;
			params.num_masks = composed.num_masks;
			params.mask_stride = composed.mask_stride;
			params.records = static_cast<const uint8_t*>(composed.d_records);
			params.record_stride = composed.record_stride;
			params.num_records = uint32_t(composed.num_records);
			params.mirror_table = composed.d_mirror_table;
			params.mirror_axis = composed.mirror_axis;
			cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
			return launch_clearing_flags(context, d_out_flags, cuda_stream, entry.c_str(), entry.c_str(),
				[&] { return launch_transform_decompress_tracks(params, composed.compose, params.db_tiers != nullptr, cuda_stream); });
		}

		// Each composed decode with checks of its own and its _skinning sibling (skinning, d_inverse_bind; the matrix object kind): the checks,
		// then the composed path
		aclb200_status decompress_additive(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_additive_request* d_requests,
			uint32_t num_requests, const aclb200_options* options, uint32_t additive_format, const uint8_t* d_clip_additive_formats,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_additive_skinning" : "decompress_tracks_additive";
			if (num_requests > 0x7FFFFFFFu)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": more than 2^31 - 1 pairs");
			if (additive_format > ACLB200_ADDITIVE_ADDITIVE1)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": additive_format out of range");
			// pair r is the two requests 2r (base) and 2r + 1 (additive) of the plain decode
			static_assert(sizeof(aclb200_additive_request) == 2 * sizeof(aclb200_request), "an additive request is two requests back to back");
			const Composed composed = { what, k_pair_unfit, k_compose_additive, 2, 0.0f, nullptr, additive_format, d_clip_additive_formats };
			return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}

		aclb200_status decompress_blend(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_blend_request* d_requests,
			uint32_t num_requests, const aclb200_options* options, float weight, const float* d_weights,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_blend_skinning" : "decompress_tracks_blend";
			if (num_requests > 0x7FFFFFFFu)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": more than 2^31 - 1 pairs");
			// pair r is the two requests 2r (from) and 2r + 1 (to) of the plain decode, the layout of aclb200_additive_request
			static_assert(sizeof(aclb200_blend_request) == 2 * sizeof(aclb200_request) && offsetof(aclb200_blend_request, to) == sizeof(aclb200_request),
				"a blend request is two requests back to back");
			const Composed composed = { what, k_pair_unfit, k_compose_blend, 2, weight, d_weights };
			return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}

		aclb200_status decompress_layered(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_layer* d_layers, uint32_t num_poses,
			uint32_t num_layers, const aclb200_options* options, uint32_t additive_format, const uint8_t* d_clip_additive_formats,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_layered_skinning" : "decompress_tracks_layered";
			const aclb200_status status = check_layers(context, num_poses, num_layers, additive_format, what);
			if (status != ACLB200_OK)
				return status;
			// stack r is the requests r L .. r L + L - 1 of the launch, read as layer records by the kernel
			static_assert(sizeof(aclb200_layer) == 16 && offsetof(aclb200_layer, pose) == 0, "a layer is a request, its op and its weight");
			const Composed composed = { what, k_layers_unfit, k_compose_layers, num_layers, 0.0f, nullptr, additive_format, d_clip_additive_formats };
			return decompress_composed(context, clipset, d_layers, num_poses, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}

		aclb200_status decompress_layered_masked(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_layer* d_layers,
			const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers, const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride,
			const aclb200_options* options, uint32_t additive_format, const uint8_t* d_clip_additive_formats,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_layered_masked_skinning" : "decompress_tracks_layered_masked";
			Composed composed = { what, k_layers_unfit, k_compose_layers_masked, num_layers, 0.0f, nullptr, additive_format, d_clip_additive_formats };
			aclb200_status status = check_layers(context, num_poses, num_layers, additive_format, what);
			if (status == ACLB200_OK)
				status = check_layer_masks(context, clipset, d_layer_masks, d_bone_masks, num_masks, mask_stride, what, composed);
			if (status != ACLB200_OK)
				return status;
			return decompress_composed(context, clipset, d_layers, num_poses, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}

		// the inertialized decode and its _skinning sibling: the record checks, then the composed path (requests are 20 byte records)
		aclb200_status decompress_inertialized(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_inertialized_request* d_requests,
			uint32_t num_requests, const aclb200_options* options, const void* d_records, uint64_t num_records, uint64_t record_stride_bytes,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_inertialized_skinning" : "decompress_tracks_inertialized";
			if (context == nullptr || clipset == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
			if (num_records >= uint64_t(ACLB200_NO_INERTIALIZATION))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": num_records must be below 2^32 - 1");
			if (num_records != 0 && d_records == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": null record pointer");
			static_assert(sizeof(aclb200_inertialized_request) == 20 && offsetof(aclb200_inertialized_request, inertialization) == 8,
				"an inertialized request is a request and its inertialization, five words");
			Composed composed = { what, k_pose_unfit, k_compose_inertialize, 1 };
			composed.record_stride = record_stride_bytes;
			const aclb200_status status = check_records(context, num_records != 0 ? d_records : nullptr, clipset->info.max_tracks,
				composed.record_stride, what);
			if (status != ACLB200_OK)
				return status;
			composed.d_records = d_records;
			composed.num_records = num_records;
			return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}

		// the mirrored decode and its _skinning sibling: the axis and table checks, then the composed path (requests are 12 byte records)
		aclb200_status decompress_mirrored(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_mirrored_request* d_requests,
			uint32_t num_requests, const aclb200_options* options, const aclb200_mirror_entry* d_mirror_table, uint32_t axis,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, bool skinning, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags, void* stream)
		{
			const char* what = skinning ? "decompress_tracks_mirrored_skinning" : "decompress_tracks_mirrored";
			if (context == nullptr || clipset == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
			const aclb200_status status = check_mirror(context, d_mirror_table, axis, num_requests != 0, what);
			if (status != ACLB200_OK)
				return status;
			static_assert(sizeof(aclb200_mirrored_request) == 12 && offsetof(aclb200_mirrored_request, mirrored) == 8,
				"a mirrored request is a request and its flag, three words");
			Composed composed = { what, k_pose_unfit, k_compose_mirror, 1 };
			composed.d_mirror_table = d_mirror_table;
			composed.mirror_axis = axis;
			return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
				skinning, d_inverse_bind, d_out, d_out_flags, stream);
		}
	}
}

using namespace aclb200;

extern "C"
{
	const char* aclb200_version_string(void)
	{
		return "aclb200 0.17 (sm_90a; ACL compressed_tracks v02_00_00..v02_01_00)";
	}

	const char* aclb200_status_string(aclb200_status status)
	{
		switch (status)
		{
		case ACLB200_OK: return "ok";
		case ACLB200_ERR_INVALID_ARGUMENT: return "invalid argument";
		case ACLB200_ERR_INVALID_CLIP: return "invalid compressed_tracks buffer";
		case ACLB200_ERR_UNSUPPORTED: return "unsupported clip";
		case ACLB200_ERR_NO_DEVICE: return "no CUDA device";
		case ACLB200_ERR_CUDA: return "CUDA error";
		case ACLB200_ERR_OUT_OF_MEMORY: return "out of device memory";
		default: return "unknown status";
		}
	}

	void aclb200_default_options(aclb200_options* options)
	{
		if (options == nullptr)
			return;
		std::memset(options, 0, sizeof(*options));
		options->struct_size = sizeof(aclb200_options);
		options->rounding_policy = ACLB200_ROUND_NONE;
		options->looping_policy = ACLB200_LOOP_AS_COMPRESSED;
		options->normalization = ACLB200_NORMALIZE_LERP_ONLY;		// default_transform_decompression_settings, decompression_settings.h:226
		options->per_track_rounding = 0;							// :231
		options->wrapping = 1;										// :153
		options->clamp_sample_time = 1;								// :80
		options->multiple_rotation_formats = 0;						// :219
		options->default_rotation_mode = ACLB200_DEFAULT_CONSTANT;	// track_writer.h:170-172
		options->default_translation_mode = ACLB200_DEFAULT_CONSTANT;
		options->default_scale_mode = ACLB200_DEFAULT_LEGACY;
		options->constant_defaults[3] = 1.0f;						// :174-176
		options->constant_defaults[8] = options->constant_defaults[9] = options->constant_defaults[10] = 1.0f;
		options->output_layout = ACLB200_LAYOUT_QVV48;
		options->math_mode = ACLB200_MATH_EXACT;
	}

	aclb200_status aclb200_create(int device, aclb200_context** out_context)
	{
		if (out_context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_context = nullptr;
		int device_count = 0;
		if (cudaGetDeviceCount(&device_count) != cudaSuccess || device_count == 0)
			return ACLB200_ERR_NO_DEVICE;		// no CPU fallback exists
		if (device < 0 || device >= device_count)
			return ACLB200_ERR_INVALID_ARGUMENT;
		cudaDeviceProp prop;
		if (cudaGetDeviceProperties(&prop, device) != cudaSuccess)
			return ACLB200_ERR_CUDA;

		aclb200_context* context = new (std::nothrow) aclb200_context();
		if (context == nullptr)
			return ACLB200_ERR_OUT_OF_MEMORY;
		context->device = device;
		context->num_sms = prop.multiProcessorCount;
		context->max_dynamic_smem = int(prop.sharedMemPerBlockOptin);
		if (prop.major != 9 || prop.minor != 0 || cudaSetDevice(device) != cudaSuccess || configure_kernels(context->max_dynamic_smem) != cudaSuccess
			|| configure_bones_kernels(context->max_dynamic_smem) != cudaSuccess || configure_features_kernels(context->max_dynamic_smem) != cudaSuccess
			|| configure_feature_search_kernels() != cudaSuccess)
		{
			// the kernels are compiled for sm_90a only, which runs on compute capability 9.0 and nothing else
			delete context;
			return ACLB200_ERR_NO_DEVICE;
		}
		*out_context = context;
		return ACLB200_OK;
	}

	void aclb200_destroy(aclb200_context* context)
	{
		if (context == nullptr)
			return;
		cudaSetDevice(context->device);
		cudaFree(context->d_scratch_requests);
		cudaFree(context->d_scratch_out);
		cudaFree(context->d_error_scratch);
		if (context->error_scratch_done != nullptr)
			cudaEventDestroy(context->error_scratch_done);
		if (context->host_stream != nullptr)
			cudaStreamDestroy(context->host_stream);
		if (context->copy_stream != nullptr)
			cudaStreamDestroy(context->copy_stream);
		for (cudaEvent_t event : context->chunk_done)
			if (event != nullptr)
				cudaEventDestroy(event);
		delete context;
	}

	const char* aclb200_last_error(const aclb200_context* context)
	{
		return context != nullptr ? context->last_error.c_str() : "null context";
	}

	aclb200_status aclb200_upload_clips(aclb200_context* context, const void* const* blobs, const uint32_t* sizes, uint32_t num_clips,
		uint32_t check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip)
	{
		if (blobs == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "upload_clips: null blob array");
		return build_clipset(context, [blobs](uint32_t clip) { return static_cast<const uint8_t*>(blobs[clip]); }, sizes, num_clips,
			check_hash != 0, out_clipset, out_failed_clip);
	}

	aclb200_status aclb200_upload_clips_packed(aclb200_context* context, const void* buffer, const uint64_t* offsets, const uint32_t* sizes,
		uint32_t num_clips, uint32_t check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip)
	{
		if (buffer == nullptr || offsets == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "upload_clips_packed: null buffer / offsets");
		const uint8_t* base = static_cast<const uint8_t*>(buffer);
		return build_clipset(context, [base, offsets](uint32_t clip) { return base + offsets[clip]; }, sizes, num_clips,
			check_hash != 0, out_clipset, out_failed_clip);
	}

	void aclb200_release_clipset(aclb200_context* context, aclb200_clipset* clipset)
	{
		if (clipset == nullptr)
			return;
		cudaSetDevice(clipset->device);
		release_base_poses(clipset);
		cudaFree(clipset->d_db_first_segment);
		cudaFree(clipset->d_data);
		cudaFree(clipset->d_clips);
		delete clipset;
		(void)context;
	}

	aclb200_status aclb200_clipset_get_info(const aclb200_clipset* clipset, aclb200_clipset_info* out_info)
	{
		if (clipset == nullptr || out_info == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_info = clipset->info;
		return ACLB200_OK;
	}

	aclb200_status aclb200_clipset_get_clip_info(const aclb200_clipset* clipset, uint32_t clip, aclb200_clip_info* out_info)
	{
		if (clipset == nullptr || out_info == nullptr || clip >= clipset->info.num_clips)
			return ACLB200_ERR_INVALID_ARGUMENT;
		const ClipDesc& desc = clipset->host_clips[clip];
		out_info->num_tracks = desc.num_tracks;
		out_info->num_samples = desc.num_samples;
		out_info->sample_rate = desc.sample_rate;
		out_info->looping_policy = clipset->host_looping[clip];
		out_info->duration = out_info->looping_policy == ACLB200_LOOP_WRAP ? desc.duration_wrap : desc.duration_clamp;
		out_info->num_segments = desc.num_segments;
		out_info->hash = desc.hash;
		out_info->size = desc.size;
		return ACLB200_OK;
	}

	aclb200_status aclb200_decompress_tracks(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, void* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, true, false, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		// launches that keep the caller's bytes store sub-tracks straight to global memory instead of assembling whole poses in shared memory
		const bool keeps_bytes = keeps_caller_bytes(*options);
		plan_launch(params, clipset->max_key_frame_bytes, context->max_dynamic_smem, !keeps_bytes, params.db_tiers != nullptr, k_compose_local);
		cudaSetDevice(context->device);
		// the plain and database kernels: one block per params.requests_per_block requests (kernels.cu, launch_tracks)
		aclb200_launch_info& launch = context->last_launch;
		launch = {};
		launch.num_requests = num_requests;
		launch.requests_per_block = params.requests_per_block;
		launch.num_batches = (num_requests + params.requests_per_block - 1) / params.requests_per_block;
		launch.grid_blocks = launch.num_batches;
		if (params.db_tiers != nullptr)
		{
			launch.kernel = ACLB200_KERNEL_DATABASE;
			return finish_launch(context, launch_transform_decompress_tracks(params, k_compose_local, true, static_cast<cudaStream_t>(stream)),
				"decompress_tracks (database)");
		}

		// Main path: the persistent TMA pipeline (pipeline.cu). It assembles whole poses in shared memory, so launches that must
		// leave `skipped` default sub-tracks untouched, or whose poses do not fit in shared memory, use the plain kernels instead.
		if (!keeps_bytes && clipset->max_key_frame_bytes != 0)
		{
			DecodeParams pipeline_params = params;
			if (plan_pipeline(pipeline_params, clipset->max_key_frame_bytes, context->max_dynamic_smem, context->num_sms))
			{
				const bool rows_16 = options->output_layout == ACLB200_LAYOUT_QVV48 || clipset->all_tracks_even;
				pipeline_params.out_bulk = rows_16 && ((uint64_t(reinterpret_cast<uintptr_t>(d_out)) | pipeline_params.pose_stride) & 15) == 0 ? 1u : 0u;
				pipeline_params.trace = context->d_trace;
				pipeline_params.trace_blocks = context->trace_blocks;
				pipeline_params.trace_iterations = context->trace_iterations;
				launch.kernel = ACLB200_KERNEL_PIPELINE;
				launch.requests_per_block = pipeline_params.requests_per_block;
				launch.num_batches = (num_requests + pipeline_params.requests_per_block - 1) / pipeline_params.requests_per_block;
				launch.grid_blocks = pipeline_params.grid_blocks;
				launch.out_bulk = pipeline_params.out_bulk;
				acquire_base_poses(clipset, pipeline_params, static_cast<cudaStream_t>(stream));
				const cudaError_t launched = launch_transform_pipeline(pipeline_params, options->math_mode, static_cast<cudaStream_t>(stream));
				release_base_poses_use(clipset, pipeline_params, static_cast<cudaStream_t>(stream));
				return finish_launch(context, launched, "decompress_tracks (pipeline)");
			}
		}
		launch.kernel = ACLB200_KERNEL_PLAIN;
		return finish_launch(context, launch_transform_decompress_tracks(params, k_compose_local, false, static_cast<cudaStream_t>(stream)), "decompress_tracks");
	}

	aclb200_status aclb200_decompress_tracks_object_space(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		const Composed composed = { "decompress_tracks_object_space", k_pose_unfit, k_compose_object, 1 };
		return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets, object_kind,
			false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		const Composed composed = { "decompress_tracks_skinning", k_pose_unfit, k_compose_object, 1 };
		return decompress_composed(context, clipset, d_requests, num_requests, options, composed, d_parent_indices, d_skeleton_offsets,
			ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_additive(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_additive(context, clipset, d_requests, num_requests, options, additive_format, d_clip_additive_formats, d_parent_indices,
			d_skeleton_offsets, object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_additive_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_additive(context, clipset, d_requests, num_requests, options, additive_format, d_clip_additive_formats, d_parent_indices,
			d_skeleton_offsets, ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_apply_additive_to_base(aclb200_context* context, const void* d_base_poses, const void* d_additive_poses,
		void* d_out, uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride_bytes, uint32_t additive_format,
		uint32_t* d_out_flags, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (additive_format > ACLB200_ADDITIVE_ADDITIVE1)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "apply_additive_to_base: additive_format out of range");
		if (num_poses == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_base_poses == nullptr || d_additive_poses == nullptr || d_out == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "apply_additive_to_base: null pose pointer");
		uint64_t stride = pose_stride_bytes;
		const aclb200_status status = check_qvvf_rows(context, { d_base_poses, d_additive_poses, d_out }, num_tracks, stride, "apply_additive_to_base");
		if (status != ACLB200_OK)
			return status;
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, "apply_additive_to_base", "apply_additive_to_base", [&] {
			return launch_apply_additive(static_cast<const uint8_t*>(d_base_poses), static_cast<const uint8_t*>(d_additive_poses),
				static_cast<uint8_t*>(d_out), num_poses, num_tracks, stride, additive_format, d_out_flags, context->num_sms, cuda_stream); });
	}

	aclb200_status aclb200_decompress_tracks_blend(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		float weight, const float* d_weights,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_blend(context, clipset, d_requests, num_requests, options, weight, d_weights, d_parent_indices, d_skeleton_offsets,
			object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_blend_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		float weight, const float* d_weights,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_blend(context, clipset, d_requests, num_requests, options, weight, d_weights, d_parent_indices, d_skeleton_offsets,
			ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_layered(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_layered(context, clipset, d_layers, num_poses, num_layers, options, additive_format, d_clip_additive_formats, d_parent_indices,
			d_skeleton_offsets, object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_layered_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_layered(context, clipset, d_layers, num_poses, num_layers, options, additive_format, d_clip_additive_formats, d_parent_indices,
			d_skeleton_offsets, ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_layered_masked(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers,
		const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_layered_masked(context, clipset, d_layers, d_layer_masks, num_poses, num_layers, d_bone_masks, num_masks, mask_stride, options,
			additive_format, d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_layered_masked_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers,
		const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options* options,
		uint32_t additive_format, const uint8_t* d_clip_additive_formats,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_layered_masked(context, clipset, d_layers, d_layer_masks, num_poses, num_layers, d_bone_masks, num_masks, mask_stride, options,
			additive_format, d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out,
			d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_bones(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list, const uint32_t* d_request_lists,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		const std::string what = "decompress_bones";
		const aclb200_status lists_checked = check_bone_lists(context, d_bone_lists, num_lists, bones_per_list, what);
		if (lists_checked != ACLB200_OK)
			return lists_checked;
		// make_params' pose stride check is the whole pose's, so the launch is described as a single track one and the stride of K rows
		// is checked here
		DecodeParams params;
		aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, true, true, params);
		if (status == ACLB200_OK)
			status = check_every_sub_track(context, *options, what);
		if (status == ACLB200_OK)
			status = check_object_output(context, *options, d_parent_indices, object_kind, what);
		if (status != ACLB200_OK)
			return status;
		const uint64_t rows_bytes = uint64_t(bones_per_list) * params.bone_stride;
		params.pose_stride = options->pose_stride_bytes != 0 ? options->pose_stride_bytes : rows_bytes;
		if (params.pose_stride < rows_bytes)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": pose_stride_bytes is smaller than bones_per_list rows");
		const bool database = params.db_tiers != nullptr;
		BoneQuery query = {};
		if (!plan_bones_launch(params, query, database, context->max_dynamic_smem))
			return set_error(context, ACLB200_ERR_UNSUPPORTED, what + k_pose_unfit);
		if (num_requests == 0)
			return ACLB200_OK;
		query.bone_lists = d_bone_lists;
		query.request_lists = d_request_lists;
		query.num_lists = num_lists;
		query.bones_per_list = bones_per_list;
		query.parent_indices = d_parent_indices;
		query.skeleton_offsets = d_skeleton_offsets;
		query.object_kind = object_kind;
		query.out_flags = d_out_flags;
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, what.c_str(), database ? "decompress_bones (database)" : "decompress_bones",
			[&] { return launch_decompress_bones(params, query, database, cuda_stream); });
	}

	aclb200_status aclb200_extract_root_motion(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_root_motion_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const uint32_t* d_root_tracks, void* d_out, uint32_t* d_out_flags, void* stream)
	{
		static_assert(sizeof(aclb200_root_motion_request) == 16, "a root motion request is one 16 byte load");
		const std::string what = "extract_root_motion";
		// the handles and the options struct's size before any option is read or the struct is copied
		const aclb200_status checked = check_handles_and_options(context, clipset, options);
		if (checked != ACLB200_OK)
			return checked;
		const aclb200_status samples_checked = check_root_samples(context, *options, what);
		if (samples_checked != ACLB200_OK)
			return samples_checked;
		// make_params refuses a scalar clip set, NULL pointers and a misaligned output; the rows are 48 bytes apart whatever
		// pose_stride_bytes says
		aclb200_options row_options = *options;
		row_options.pose_stride_bytes = 0;
		DecodeParams params;
		aclb200_status status = make_params(context, clipset, reinterpret_cast<const aclb200_request*>(d_requests), num_requests, &row_options, d_out,
			true, true, params);
		if (status == ACLB200_OK)
			status = check_every_sub_track(context, row_options, what);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		params.requests = nullptr;
		params.pose_stride = 48;
		const RootMotionQuery query = { d_requests, d_root_tracks, d_out_flags };
		const bool database = params.db_tiers != nullptr;
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, what.c_str(), database ? "extract_root_motion (database)" : "extract_root_motion",
			[&] { return launch_extract_root_motion(params, query, database, cuda_stream); });
	}

	aclb200_status aclb200_extract_pose_features(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_feature_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const float* offsets, uint32_t num_offsets,
		const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list, const uint32_t* d_request_lists,
		const uint32_t* d_root_tracks, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		static_assert(sizeof(aclb200_feature_request) == 12, "a feature request is three 4 byte fields");
		const std::string what = "extract_pose_features";
		// the handles and the options struct's size before any option is read
		const aclb200_status checked = check_handles_and_options(context, clipset, options);
		if (checked != ACLB200_OK)
			return checked;
		if (offsets == nullptr || num_offsets == 0 || num_offsets > ACLB200_MAX_FEATURE_OFFSETS)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": needs 1 to 8 offsets (num_offsets), offsets not NULL");
		for (uint32_t s = 0; s < num_offsets; ++s)
			if (!std::isfinite(offsets[s]))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": every offset must be finite");
		if (uint64_t(num_requests) * num_offsets > 0xFFFFFFFFull)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": num_requests * num_offsets must fit in 32 bits");
		if (d_parent_indices == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": the features are object space rows, d_parent_indices must be given");
		const aclb200_status lists_checked = check_bone_lists(context, d_bone_lists, num_lists, bones_per_list, what);
		if (lists_checked != ACLB200_OK)
			return lists_checked;
		const aclb200_status samples_checked = check_root_samples(context, *options, what);
		if (samples_checked != ACLB200_OK)
			return samples_checked;
		// make_params refuses a scalar clip set, NULL pointers and a misaligned output; the stride of S * K rows is checked here
		DecodeParams params;
		aclb200_status status = make_params(context, clipset, reinterpret_cast<const aclb200_request*>(d_requests), num_requests, options, d_out,
			true, true, params);
		if (status == ACLB200_OK)
			status = check_every_sub_track(context, *options, what);
		if (status == ACLB200_OK)
			status = check_object_output(context, *options, d_parent_indices, ACLB200_OBJECT_QVVF, what);
		if (status != ACLB200_OK)
			return status;
		const uint64_t rows_bytes = uint64_t(num_offsets) * bones_per_list * 48;
		params.pose_stride = options->pose_stride_bytes != 0 ? options->pose_stride_bytes : rows_bytes;
		if (params.pose_stride < rows_bytes)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": pose_stride_bytes is smaller than num_offsets * bones_per_list rows");
		const bool database = params.db_tiers != nullptr;
		BoneQuery query = {};
		if (!plan_features_launch(params, query, database, context->max_dynamic_smem))
			return set_error(context, ACLB200_ERR_UNSUPPORTED, what + k_pose_unfit);
		if (num_requests == 0)
			return ACLB200_OK;
		params.requests = nullptr;
		params.num_requests = num_requests * num_offsets;
		query.bone_lists = d_bone_lists;
		query.request_lists = d_request_lists;
		query.num_lists = num_lists;
		query.bones_per_list = bones_per_list;
		query.parent_indices = d_parent_indices;
		query.skeleton_offsets = d_skeleton_offsets;
		query.object_kind = ACLB200_OBJECT_QVVF;
		query.out_flags = d_out_flags;
		FeatureQuery features = {};
		features.requests = d_requests;
		features.root_tracks = d_root_tracks;
		std::memcpy(features.offsets, offsets, num_offsets * sizeof(float));
		features.num_offsets = num_offsets;
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, what.c_str(), database ? "extract_pose_features (database)" : "extract_pose_features",
			[&] { return launch_extract_pose_features(params, query, features, database, cuda_stream); });
	}

	aclb200_status aclb200_pack_pose_features(aclb200_context* context, const void* d_rows, uint32_t num_requests, uint32_t num_offsets,
		uint32_t bones_per_list, uint64_t pose_stride_bytes, const aclb200_feature_term* terms, uint32_t num_terms, const float* mean,
		const float* scale, uint32_t num_dims, float* d_out, uint32_t out_stride, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		const std::string what = "pack_pose_features";
		if (num_offsets == 0 || num_offsets > ACLB200_MAX_FEATURE_OFFSETS || bones_per_list == 0 || bones_per_list > ACLB200_MAX_QUERY_BONES)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": needs 1 to 8 offsets and 1 to 32 bones per list");
		if (num_dims == 0 || num_dims > ACLB200_MAX_FEATURE_DIMS)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": num_dims must be 1 to 64");
		if (terms == nullptr || num_terms == 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": needs at least one term");
		PackParams params = {};
		uint32_t d = 0;
		for (uint32_t t = 0; t < num_terms; ++t)
		{
			const aclb200_feature_term& term = terms[t];
			if (term.kind > ACLB200_FEATURE_VELOCITY || term.s0 >= num_offsets || term.k >= bones_per_list || term.components == 0
				|| term.components > 7 || (term.kind == ACLB200_FEATURE_VELOCITY && (term.s1 >= num_offsets || !std::isfinite(term.inv_dt)))
				|| (term.kind == ACLB200_FEATURE_DIRECTION && term.axis > 2))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": term " + std::to_string(t)
					+ " has an unknown kind, a row outside the S x K rows, an axis above 2, components outside 1..7 or a non-finite inv_dt");
			for (uint32_t c = 0; c < 3; ++c)
			{
				if ((term.components & (1u << c)) == 0)
					continue;
				if (d == num_dims)
					return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": the terms emit more than num_dims components");
				PackDim& dim = params.dims[d];
				dim.kind = term.kind;
				dim.row0 = term.s0 * bones_per_list + term.k;
				dim.row1 = term.kind == ACLB200_FEATURE_VELOCITY ? term.s1 * bones_per_list + term.k : dim.row0;
				dim.component = c;
				dim.axis = term.kind == ACLB200_FEATURE_DIRECTION ? term.axis : 0u;
				dim.inv_dt = term.kind == ACLB200_FEATURE_VELOCITY ? term.inv_dt : 1.0f;
				dim.mean = mean != nullptr ? mean[d] : 0.0f;
				dim.scale = scale != nullptr ? scale[d] : 1.0f;
				if (!std::isfinite(dim.mean) || !std::isfinite(dim.scale))
					return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": mean and scale must be finite");
				++d;
			}
		}
		if (d != num_dims)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": the terms emit fewer than num_dims components");
		const uint64_t rows_bytes = uint64_t(num_offsets) * bones_per_list * 48;
		const uint64_t pose_stride = pose_stride_bytes != 0 ? pose_stride_bytes : rows_bytes;
		if (pose_stride < rows_bytes || (pose_stride % 16) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": pose_stride_bytes must hold S * K rows and be a multiple of 16");
		if (out_stride < num_dims || (out_stride % 4) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": out_stride must be at least num_dims and a multiple of 4 floats");
		if (num_requests == 0)
			return ACLB200_OK;
		if (d_rows == nullptr || d_out == nullptr || ((reinterpret_cast<uintptr_t>(d_rows) | reinterpret_cast<uintptr_t>(d_out)) % 16) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": d_rows and d_out must be 16 byte aligned device pointers");
		params.rows = static_cast<const uint8_t*>(d_rows);
		params.pose_stride = pose_stride;
		params.out = d_out;
		params.out_stride = out_stride;
		params.num_requests = num_requests;
		params.num_dims = num_dims;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_pack_pose_features(params, static_cast<cudaStream_t>(stream)), what.c_str());
	}

	aclb200_status aclb200_search_pose_features(aclb200_context* context, const float* d_database, uint64_t num_rows, uint64_t db_stride,
		const uint32_t* d_row_tags, const float* d_query_vectors, const aclb200_search_query* d_queries, uint32_t num_queries, uint64_t q_stride,
		uint32_t num_dims, aclb200_search_result* d_results, void* stream)
	{
		static_assert(sizeof(aclb200_search_result) == 8 && offsetof(aclb200_search_result, cost) == 4,
			"a result read as a little endian uint64 is (cost bits << 32) | row");
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		const std::string what = "search_pose_features";
		if (num_dims == 0 || num_dims > ACLB200_MAX_FEATURE_DIMS)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": num_dims must be 1 to 64");
		if (db_stride < num_dims || q_stride < num_dims || (db_stride % 4) != 0 || (q_stride % 4) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": db_stride and q_stride must be at least num_dims and multiples of 4 floats");
		if (num_rows >= 0xFFFFFFFFull)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": num_rows must be below 2^32 - 1 (ACLB200_NO_ROW)");
		if (num_rows != 0 && d_database == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": null database");
		if (num_queries != 0 && (d_query_vectors == nullptr || d_queries == nullptr || d_results == nullptr))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": null query / result pointer");
		if (((reinterpret_cast<uintptr_t>(d_database) | reinterpret_cast<uintptr_t>(d_query_vectors)) % 16) != 0
			|| (reinterpret_cast<uintptr_t>(d_results) % 8) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, what + ": vectors must be 16 byte aligned, results 8 byte aligned");
		if (num_queries == 0)
			return ACLB200_OK;
		SearchParams params = {};
		params.database = d_database;
		params.query_vectors = d_query_vectors;
		params.queries = d_queries;
		params.row_tags = d_row_tags;
		params.results = d_results;
		params.num_rows = num_rows;
		params.db_stride = db_stride;
		params.q_stride = q_stride;
		params.num_queries = num_queries;
		params.num_dims = num_dims;
		cudaSetDevice(context->device);
		const aclb200_status status = finish_launch(context, launch_search_pose_features(params, context->num_sms, static_cast<cudaStream_t>(stream)),
			what.c_str());
		if (status == ACLB200_OK && num_rows != 0)
			context->launch_count++;		// the results' clear, then the search: two kernels
		return status;
	}

	aclb200_status aclb200_blend_poses(aclb200_context* context, const void* d_from_poses, const void* d_to_poses, void* d_out,
		uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride_bytes, float weight, const float* d_weights, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (num_poses == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_from_poses == nullptr || d_to_poses == nullptr || d_out == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "blend_poses: null pose pointer");
		uint64_t stride = pose_stride_bytes;
		const aclb200_status status = check_qvvf_rows(context, { d_from_poses, d_to_poses, d_out }, num_tracks, stride, "blend_poses");
		if (status != ACLB200_OK)
			return status;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_blend_poses(static_cast<const uint8_t*>(d_from_poses), static_cast<const uint8_t*>(d_to_poses),
			static_cast<uint8_t*>(d_out), num_poses, num_tracks, stride, weight, d_weights, context->num_sms, static_cast<cudaStream_t>(stream)),
			"blend_poses");
	}

	aclb200_status aclb200_begin_inertialization(aclb200_context* context, const void* d_src, const void* d_src_prev, const void* d_dst,
		const void* d_dst_prev, uint64_t num_transitions, uint32_t num_tracks, uint64_t pose_stride_bytes, float inv_dt, void* d_records,
		uint64_t record_stride_bytes, const uint32_t* d_record_slots, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (!std::isfinite(inv_dt) || inv_dt == 0.0f)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "begin_inertialization: inv_dt must be finite and not zero");
		if (num_transitions == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_src == nullptr || d_src_prev == nullptr || d_dst == nullptr || d_dst_prev == nullptr || d_records == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "begin_inertialization: null pose or record pointer");
		uint64_t stride = pose_stride_bytes;
		aclb200_status status = check_qvvf_rows(context, { d_src, d_src_prev, d_dst, d_dst_prev }, num_tracks, stride, "begin_inertialization");
		if (status != ACLB200_OK)
			return status;
		uint64_t record_stride = record_stride_bytes;
		status = check_records(context, d_records, num_tracks, record_stride, "begin_inertialization");
		if (status != ACLB200_OK)
			return status;
		if (reinterpret_cast<uintptr_t>(d_record_slots) % 4 != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "begin_inertialization: record slots must be 4 byte aligned");
		InertializationCapture capture = {};
		capture.src = static_cast<const uint8_t*>(d_src);
		capture.src_prev = static_cast<const uint8_t*>(d_src_prev);
		capture.dst = static_cast<const uint8_t*>(d_dst);
		capture.dst_prev = static_cast<const uint8_t*>(d_dst_prev);
		capture.records = static_cast<uint8_t*>(d_records);
		capture.record_slots = d_record_slots;
		capture.num_transitions = num_transitions;
		capture.pose_stride = stride;
		capture.record_stride = record_stride;
		capture.num_tracks = num_tracks;
		capture.inv_dt = inv_dt;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_begin_inertialization(capture, context->num_sms, static_cast<cudaStream_t>(stream)), "begin_inertialization");
	}

	aclb200_status aclb200_inertialize_poses(aclb200_context* context, const void* d_poses, void* d_out, uint64_t num_poses,
		uint32_t num_tracks, uint64_t pose_stride_bytes, const aclb200_inertialization* d_inertializations, const void* d_records,
		uint64_t num_records, uint64_t record_stride_bytes, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (num_records >= uint64_t(ACLB200_NO_INERTIALIZATION))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "inertialize_poses: num_records must be below 2^32 - 1");
		uint64_t record_stride = record_stride_bytes;
		aclb200_status status = check_records(context, num_records != 0 ? d_records : nullptr, num_tracks, record_stride, "inertialize_poses");
		if (status != ACLB200_OK)
			return status;
		if (num_poses == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_poses == nullptr || d_out == nullptr || d_inertializations == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "inertialize_poses: null pose or inertialization pointer");
		if (reinterpret_cast<uintptr_t>(d_inertializations) % 4 != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "inertialize_poses: inertializations must be 4 byte aligned");
		if (num_records != 0 && d_records == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "inertialize_poses: null record pointer");
		uint64_t stride = pose_stride_bytes;
		status = check_qvvf_rows(context, { d_poses, d_out }, num_tracks, stride, "inertialize_poses");
		if (status != ACLB200_OK)
			return status;
		InertializationApply apply = {};
		apply.poses = static_cast<const uint8_t*>(d_poses);
		apply.out = static_cast<uint8_t*>(d_out);
		apply.inertializations = d_inertializations;
		apply.records = static_cast<const uint8_t*>(d_records);
		apply.num_poses = num_poses;
		apply.pose_stride = stride;
		apply.record_stride = record_stride;
		apply.num_records = num_records;
		apply.num_tracks = num_tracks;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_inertialize_poses(apply, context->num_sms, static_cast<cudaStream_t>(stream)), "inertialize_poses");
	}

	aclb200_status aclb200_decompress_tracks_inertialized(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_inertialized_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const void* d_records, uint64_t num_records, uint64_t record_stride_bytes,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_inertialized(context, clipset, d_requests, num_requests, options, d_records, num_records, record_stride_bytes,
			d_parent_indices, d_skeleton_offsets, object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_inertialized_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_inertialized_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const void* d_records, uint64_t num_records, uint64_t record_stride_bytes,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_inertialized(context, clipset, d_requests, num_requests, options, d_records, num_records, record_stride_bytes,
			d_parent_indices, d_skeleton_offsets, ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_mirror_poses(aclb200_context* context, const void* d_poses, void* d_out, uint64_t num_poses, uint32_t num_rows,
		uint64_t pose_stride_bytes, const uint32_t* d_mirrored, const aclb200_mirror_entry* d_table, uint32_t axis, uint32_t* d_out_flags,
		void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		const bool work = num_poses != 0 && num_rows != 0;
		aclb200_status status = check_mirror(context, d_table, axis, work, "mirror_poses");
		if (status != ACLB200_OK)
			return status;
		if (!work)
			return ACLB200_OK;
		if (d_poses == nullptr || d_out == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "mirror_poses: null pose pointer");
		if (reinterpret_cast<uintptr_t>(d_mirrored) % 4 != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "mirror_poses: d_mirrored must be 4 byte aligned");
		uint64_t stride = pose_stride_bytes;
		status = check_qvvf_rows(context, { d_poses, d_out }, num_rows, stride, "mirror_poses");
		if (status != ACLB200_OK)
			return status;
		MirrorApply apply = {};
		apply.poses = static_cast<const uint8_t*>(d_poses);
		apply.out = static_cast<uint8_t*>(d_out);
		apply.mirrored = d_mirrored;
		apply.table = d_table;
		apply.flags = d_out_flags;
		apply.num_poses = num_poses;
		apply.pose_stride = stride;
		apply.num_rows = num_rows;
		apply.axis = axis;
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, "mirror_poses", "mirror_poses",
			[&] { return launch_mirror_poses(apply, context->num_sms, cuda_stream); });
	}

	aclb200_status aclb200_decompress_tracks_mirrored(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const aclb200_mirror_entry* d_mirror_table, uint32_t axis,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_mirrored(context, clipset, d_requests, num_requests, options, d_mirror_table, axis, d_parent_indices, d_skeleton_offsets,
			object_kind, false, nullptr, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_decompress_tracks_mirrored_skinning(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options* options,
		const aclb200_mirror_entry* d_mirror_table, uint32_t axis,
		const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
		void* d_out, uint32_t* d_out_flags, void* stream)
	{
		return decompress_mirrored(context, clipset, d_requests, num_requests, options, d_mirror_table, axis, d_parent_indices, d_skeleton_offsets,
			ACLB200_OBJECT_MATRIX3X4F, true, d_inverse_bind, d_out, d_out_flags, stream);
	}

	aclb200_status aclb200_local_to_skinning(aclb200_context* context, const void* d_local_poses, void* d_out, uint64_t num_poses, uint32_t num_tracks,
		uint64_t pose_stride_bytes, const uint32_t* d_parent_indices, const float* d_inverse_bind, uint32_t* d_out_flags, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (num_poses == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_local_poses == nullptr || d_out == nullptr || d_parent_indices == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "local_to_skinning: null pose / parent pointer");
		uint64_t stride = pose_stride_bytes;
		aclb200_status status = check_qvvf_rows(context, { d_local_poses, d_out }, num_tracks, stride, "local_to_skinning");
		if (status == ACLB200_OK)
			status = check_inverse_binds(context, d_inverse_bind, "local_to_skinning");
		if (status != ACLB200_OK)
			return status;
		const uint32_t warps = local_to_skinning_warps(num_tracks, context->max_dynamic_smem);
		if (warps == 0)
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "local_to_skinning: one pose does not fit in a block's shared memory");
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		return launch_clearing_flags(context, d_out_flags, cuda_stream, "local_to_skinning", "local_to_skinning", [&] {
			return launch_local_to_skinning(static_cast<const uint8_t*>(d_local_poses), static_cast<uint8_t*>(d_out), num_poses, num_tracks, stride,
				d_parent_indices, d_inverse_bind, d_out_flags, warps, context->num_sms, cuda_stream); });
	}

	aclb200_status aclb200_decompress_track(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, const uint32_t* d_track_indices, uint32_t num_requests,
		const aclb200_options* options, void* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, true, true, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		if (d_track_indices == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null track index pointer");
		params.track_indices = d_track_indices;
		cudaSetDevice(context->device);
		const bool database = params.db_tiers != nullptr;
		return finish_launch(context, launch_transform_decompress_track(params, database, static_cast<cudaStream_t>(stream)),
			database ? "decompress_track (database)" : "decompress_track");
	}

	aclb200_status aclb200_scalar_decompress_tracks(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, void* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, false, false, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		cudaSetDevice(context->device);
		plan_scalar_launch(params, clipset->max_key_frame_bytes);
		return finish_launch(context, launch_scalar_decompress_tracks(params, static_cast<cudaStream_t>(stream)), "scalar_decompress_tracks");
	}

	aclb200_status aclb200_scalar_decompress_track(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, const uint32_t* d_track_indices, uint32_t num_requests,
		const aclb200_options* options, void* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, false, true, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		if (d_track_indices == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null track index pointer");
		params.track_indices = d_track_indices;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_scalar_decompress_track(params, static_cast<cudaStream_t>(stream)), "scalar_decompress_track");
	}

	aclb200_status aclb200_decompress_tracks_host(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* requests, uint32_t num_requests, const aclb200_options* options, void* out, size_t out_bytes)
	{
		if (context == nullptr || clipset == nullptr || options == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
		if (num_requests == 0)
			return ACLB200_OK;
		if (requests == nullptr || out == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null request / output pointer");

		const bool is_transform = clipset->info.track_type == ACLB200_TRACK_QVVF;
		const uint32_t bone_stride = is_transform ? (options->output_layout == ACLB200_LAYOUT_QVV48 ? 48u : 40u) : scalar_components(clipset->info.track_type) * 4u;
		const uint64_t pose_stride = options->pose_stride_bytes != 0 ? options->pose_stride_bytes : uint64_t(clipset->info.max_tracks) * bone_stride;
		const size_t needed_out = size_t(pose_stride) * num_requests;
		if (out_bytes < needed_out)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "output buffer too small");
		const size_t needed_requests = sizeof(aclb200_request) * size_t(num_requests);

		cudaError_t error = cudaSetDevice(context->device);
		if (error == cudaSuccess && context->host_stream == nullptr)
			error = cudaStreamCreateWithFlags(&context->host_stream, cudaStreamNonBlocking);
		if (error == cudaSuccess && context->scratch_requests_bytes < needed_requests)
		{
			cudaFree(context->d_scratch_requests);
			context->d_scratch_requests = nullptr;
			context->scratch_requests_bytes = 0;
			error = cudaMalloc(&context->d_scratch_requests, needed_requests);
			if (error == cudaSuccess) context->scratch_requests_bytes = needed_requests;
		}
		if (error == cudaSuccess && context->scratch_out_bytes < needed_out)
		{
			cudaFree(context->d_scratch_out);
			context->d_scratch_out = nullptr;
			context->scratch_out_bytes = 0;
			error = cudaMalloc(&context->d_scratch_out, needed_out);
			if (error == cudaSuccess) context->scratch_out_bytes = needed_out;
		}
		if (error != cudaSuccess)
			return check_cuda(context, error, "decompress_tracks_host: scratch allocation");

		cudaStream_t stream = context->host_stream;
		if (context->copy_stream == nullptr)
			error = cudaStreamCreateWithFlags(&context->copy_stream, cudaStreamNonBlocking);
		for (int i = 0; i < 2 && error == cudaSuccess; ++i)
			if (context->chunk_done[i] == nullptr)
				error = cudaEventCreateWithFlags(&context->chunk_done[i], cudaEventDisableTiming);
		if (error != cudaSuccess)
			return check_cuda(context, error, "decompress_tracks_host: streams");

		// `skipped` default sub-tracks keep what the caller's buffer held: bring the buffer in first in that case
		const bool keeps_input = is_transform && keeps_caller_bytes(*options);
		// Rows no request writes (clips shorter than the widest one, requests naming a clip outside the set) read as zero. Clearing the
		// scratch costs a pass over it, so it only happens when such rows can exist.
		bool needs_clear = !keeps_input && (clipset->info.min_tracks != clipset->info.max_tracks || pose_stride != uint64_t(clipset->info.max_tracks) * bone_stride);
		if (!keeps_input && !needs_clear)
			for (uint32_t r = 0; r < num_requests && !needs_clear; ++r)
				needs_clear = requests[r].clip >= clipset->info.num_clips;

		error = cudaMemcpyAsync(context->d_scratch_requests, requests, needed_requests, cudaMemcpyHostToDevice, stream);
		if (error == cudaSuccess && keeps_input)
			error = cudaMemcpyAsync(context->d_scratch_out, out, needed_out, cudaMemcpyHostToDevice, stream);
		else if (error == cudaSuccess && needs_clear)
			error = cudaMemsetAsync(context->d_scratch_out, 0, needed_out, stream);
		if (error != cudaSuccess)
			return check_cuda(context, error, "decompress_tracks_host: upload");

		// Decode in a few chunks on one stream while the previous chunk's poses cross PCIe on another: the copy is the long pole
		// (tens of milliseconds per GB against well under a millisecond of decode), so it starts as early as possible and never waits
		// for the whole batch.
		const uint32_t num_chunks = num_requests >= 65536 ? 8u : (num_requests >= 4096 ? 2u : 1u);
		const aclb200_request* d_requests = static_cast<const aclb200_request*>(context->d_scratch_requests);
		uint8_t* d_out = static_cast<uint8_t*>(context->d_scratch_out);
		for (uint32_t chunk = 0; chunk < num_chunks; ++chunk)
		{
			const uint32_t first = uint32_t(uint64_t(num_requests) * chunk / num_chunks);
			const uint32_t last = uint32_t(uint64_t(num_requests) * (chunk + 1) / num_chunks);
			if (first == last)
				continue;
			uint8_t* d_chunk = d_out + size_t(first) * pose_stride;
			// a chunk's requests start at `first`: so do their policy pairs
			aclb200_options chunk_options = *options;
			if (chunk_options.d_request_policies != nullptr)
				chunk_options.d_request_policies += size_t(first) * 2;
			const aclb200_status status = is_transform
				? aclb200_decompress_tracks(context, clipset, d_requests + first, last - first, &chunk_options, d_chunk, stream)
				: aclb200_scalar_decompress_tracks(context, clipset, d_requests + first, last - first, &chunk_options, d_chunk, stream);
			if (status != ACLB200_OK)
			{
				cudaStreamSynchronize(stream);
				cudaStreamSynchronize(context->copy_stream);
				return status;
			}
			cudaEvent_t done = context->chunk_done[chunk & 1];
			error = cudaEventRecord(done, stream);
			if (error == cudaSuccess) error = cudaStreamWaitEvent(context->copy_stream, done, 0);
			if (error == cudaSuccess)
				error = cudaMemcpyAsync(static_cast<uint8_t*>(out) + size_t(first) * pose_stride, d_chunk, size_t(last - first) * pose_stride, cudaMemcpyDeviceToHost, context->copy_stream);
			if (error != cudaSuccess)
				break;
		}
		const cudaError_t sync_decode = cudaStreamSynchronize(stream);
		const cudaError_t sync_copy = cudaStreamSynchronize(context->copy_stream);
		if (error == cudaSuccess) error = sync_decode;
		if (error == cudaSuccess) error = sync_copy;
		return check_cuda(context, error, "decompress_tracks_host: download");
	}

	aclb200_status aclb200_debug_seek(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, aclb200_seek_state* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, true, true, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		if (params.db_tiers != nullptr)
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "debug_seek: the clip set's database has chunks streamed in");
		cudaSetDevice(context->device);
		return finish_launch(context, launch_transform_debug_seek(params, d_out, static_cast<cudaStream_t>(stream)), "debug_seek");
	}

	aclb200_status aclb200_debug_unpack(aclb200_context* context, const aclb200_clipset* clipset,
		const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options* options, uint32_t which,
		uint32_t max_animated_sub_tracks, uint32_t* d_out, void* stream)
	{
		DecodeParams params;
		const aclb200_status status = make_params(context, clipset, d_requests, num_requests, options, d_out, true, true, params);
		if (status != ACLB200_OK || num_requests == 0)
			return status;
		if (which > 1)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "key frame selector must be 0 or 1");
		if (params.db_tiers != nullptr)
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "debug_unpack: the clip set's database has chunks streamed in");
		params.debug_which = which;
		params.debug_max_sub_tracks = max_animated_sub_tracks;
		cudaSetDevice(context->device);
		return finish_launch(context, launch_transform_debug_unpack(params, d_out, static_cast<cudaStream_t>(stream)), "debug_unpack");
	}

	aclb200_status aclb200_debug_set_trace(aclb200_context* context, void* d_trace, uint32_t num_blocks, uint32_t num_iterations)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		context->d_trace = static_cast<unsigned long long*>(d_trace);
		context->trace_blocks = d_trace != nullptr ? num_blocks : 0;
		context->trace_iterations = d_trace != nullptr ? num_iterations : 0;
		return ACLB200_OK;
	}

	aclb200_status aclb200_debug_last_launch(const aclb200_context* context, aclb200_launch_info* out_info)
	{
		if (context == nullptr || out_info == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_info = context->last_launch;
		return ACLB200_OK;
	}

	aclb200_status aclb200_device_malloc(aclb200_context* context, size_t bytes, void** out_device_pointer)
	{
		if (context == nullptr || out_device_pointer == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_device_pointer = nullptr;
		cudaSetDevice(context->device);
		return check_cuda(context, cudaMalloc(out_device_pointer, bytes == 0 ? 1 : bytes), "device_malloc");
	}

	void aclb200_device_free(aclb200_context* context, void* device_pointer)
	{
		if (context == nullptr || device_pointer == nullptr)
			return;
		cudaSetDevice(context->device);
		cudaFree(device_pointer);
	}

	aclb200_status aclb200_copy_to_device(aclb200_context* context, void* device_destination, const void* host_source, size_t bytes)
	{
		if (context == nullptr || (bytes != 0 && (device_destination == nullptr || host_source == nullptr)))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "copy_to_device: null pointer");
		cudaSetDevice(context->device);
		return check_cuda(context, cudaMemcpy(device_destination, host_source, bytes, cudaMemcpyHostToDevice), "copy_to_device");
	}

	aclb200_status aclb200_copy_to_host(aclb200_context* context, void* host_destination, const void* device_source, size_t bytes)
	{
		if (context == nullptr || (bytes != 0 && (host_destination == nullptr || device_source == nullptr)))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "copy_to_host: null pointer");
		cudaSetDevice(context->device);
		return check_cuda(context, cudaMemcpy(host_destination, device_source, bytes, cudaMemcpyDeviceToHost), "copy_to_host");
	}

	uint64_t aclb200_launch_count(const aclb200_context* context)
	{
		return context != nullptr ? context->launch_count : 0;
	}
}
