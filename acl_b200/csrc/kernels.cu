// acl_b200/csrc/kernels.cu -- sm_90a kernels of the batched ACL decompression path.
//
// One launch decodes `num_requests` (clip, sample_time) requests == that many
//   context.seek(t, policy); context.decompress_tracks(writer);
// sequences of the reference (includes/acl/decompression/decompress.h:147-166). The kernel is fused: the seek
// (key frame / segment lookup, seek_v0, decompression/impl/decompression.transform.h:206-563), the variable bit
// rate unpack (unpack_animated_quat / unpack_animated_vector3, animated_track_cache.transform.h:515-687,871-990),
// the segment + clip range expansion (:157-350,391-466), the quaternion W reconstruction, the key frame
// interpolation and normalisation (math/quatf.h:135-211) all happen in one pass, and every pose byte is written once.
//
// Work decomposition (not the reference's: the CPU walks nine serial passes with running cursors):
//   thread block = `requests_per_block` whole requests.
//     phase 1  one thread per request runs the seek, stores the request state in shared memory and asks the TMA unit
//              (cp.async.bulk + mbarrier) to stage the request's two key frames -- a few hundred contiguous bytes of the
//              packed segment stream each -- in shared memory.
//     phase 2  while those copies fly: one thread per (request, bone) writes the constant and default sub-tracks.
//     phase 3  one thread per (request, animated rotation sub-track): unpack both key frames from shared memory, expand,
//              reconstruct W, lerp, normalise, store the quaternion.
//     phase 4  one thread per (request, animated translation / scale sub-track).
//   The passes are compacted per sub-track class, so warps do not diverge between animated and constant bones; the clip
//   image built at upload (layout.h) gives every thread its operands with 16 byte loads and no dependency on other threads.
//
// Arithmetic contract (EXACT mode): every float operation is an IEEE-754 round-to-nearest mul/add/sub/sqrt/rcp
// issued in the reference's order through __fmul_rn/__fadd_rn/... intrinsics, which nvcc never contracts into FMAs
// (the reference never fuses either: external/rtm/includes/rtm/impl/macros.vector4.impl.h:67,93,122). The results
// are bit-identical to the reference's SSE2/AVX/scalar builds for decompress_tracks.
#include "device_common.cuh"
#include "object_space.cuh"

#include <type_traits>

namespace aclb200
{
	using namespace dev;

	namespace
	{
		// The layered decode keeps one slot per request beside the request states. op: the layer's ACLB200_LAYER_*, k_layer_base for the
		// first layer of its stack that is not OFF, k_layer_unknown for an op above ACLB200_LAYER_ADDITIVE (or, masked decode, a mask index
		// at or above num_masks), in the low k_layer_op_bits; masked decode: above them the layer's mask index + 1 (0: no mask; only BLEND
		// and ADDITIVE layers above the base carry one); weight: its weight.
		// stack_base of slot i: the block-local request whose row holds stack i's running pose, k_no_base when stack i writes nothing.
		// num_stacks of slot 0: the stacks of the block (read from here after the decode, so that no register holds it through the fold).
		struct alignas(16) LayerSlot
		{
			uint32_t op;
			float    weight;
			uint32_t stack_base;
			uint32_t num_stacks;
		};
		static_assert(sizeof(LayerSlot) == 16, "a layer slot is 16 bytes beside each request state");

		// The inertialized decode keeps each request's aclb200_inertialization in the same 16 byte slot beside its state
		struct alignas(16) InertializationSlot
		{
			uint32_t record;
			float    elapsed;
			float    halflife;
			uint32_t unused;
		};
		static_assert(sizeof(InertializationSlot) == sizeof(LayerSlot), "an inertialization slot takes a layer slot's place");

		// The mirrored decode keeps each request's `mirrored` word in the same 16 byte slot
		struct alignas(16) MirrorSlot
		{
			uint32_t mirrored;
			uint32_t unused[3];
		};
		static_assert(sizeof(MirrorSlot) == sizeof(LayerSlot), "a mirror slot takes a layer slot's place");
		constexpr uint32_t k_layer_base = 3, k_layer_unknown = 4, k_no_base = 0xFFFFFFFFu;
		constexpr uint32_t k_layer_op_mask = (1u << k_layer_op_bits) - 1;

		// The track_writer default pose as one pose row, [QVV40][scale one]: identity rotation, zero translation, scale 0 or 1 (the clip's
		// k_clip_default_scale_one), QVV48 (rotation, translation + 0, scale + 0) and QVV40 (rotation, translation, scale) rows. It is the
		// identity of every additive format: a weighted ADDITIVE layer lerps its row from it.
		__device__ __align__(16) const float k_writer_default_rows[2][2][12] = {
			{ { 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0 }, { 0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0 } },
			{ { 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0 }, { 0, 0, 0, 1, 0, 0, 0, 1, 1, 1, 0, 0 } },
		};

		// ---------------------------------------------------------------------------------------------------
		// kernels
		// ---------------------------------------------------------------------------------------------------
		// STAGED    : the two key frames of every request are staged in shared memory by the TMA unit (else read from global memory)
		// OUT_STAGED: poses are assembled in shared memory and written out with full-line coalesced 16 byte stores (else every
		//             phase stores its sub-tracks straight to global memory: needed when `skipped` default sub-tracks must keep
		//             what the caller's buffer holds, or when a pose does not fit in shared memory)
		// DB        : the clip set's bound database has chunks streamed in: key frames may come from its tier buffers
		// COMPOSE   : every mode but k_compose_local needs OUT_STAGED.
		//             k_compose_object: the staged poses are taken to object space before they leave (aclb200_decompress_tracks_object_space, QVV48)
		//             k_compose_additive, k_compose_blend: requests 2r and 2r + 1 are the two halves of pair r (whole pairs per block); phase 4c
		//             combines the two rows into row 2r, which is taken to object space when parents are given (p.parent_indices, a run-time
		//             branch) and leaves as output r.
		//             additive (aclb200_decompress_tracks_additive): base and additive half; the additive half takes the track_writer defaults.
		//             blend (aclb200_decompress_tracks_blend): from and to half, both full poses; row 2r becomes rtm::qvv_lerp(from, to, weight).
		//             The object kind k_object_skinning (the _skinning entry points) is a run-time value like the other kinds: the matrix walk,
		//             then the skinning step of object_space.cuh on the whole pose.
		//             k_compose_layers (aclb200_decompress_tracks_layered): requests r L .. r L + L - 1 are the layers of stack r (L = p.num_layers
		//             at run time, whole stacks per block), read as 16 byte aclb200_layer records. An OFF layer is not sought. Phase 4c folds the
		//             later layers into the base row (the first layer that is not OFF) with the pair modes' blend_row / apply_additive_row;
		//             phases 4b and 5 take the base row.
		//             k_compose_layers_masked (aclb200_decompress_tracks_layered_masked): the layered mode where each layer may carry a bone
		//             mask (its weight times mask[bone], skipped where the mask is +-0) and ADDITIVE layers take their weight. A mode of its
		//             own rather than a run-time switch of k_compose_layers: the switch made the unmasked fold 1.4 % slower on C2.
		//             k_compose_inertialize (aclb200_decompress_tracks_inertialized): requests are 20 byte aclb200_inertialized_request
		//             records; a request whose record is at or above p.num_records is not sought (it writes nothing). Phase 4c decays the
		//             record's offset onto each bone's row in place (obj::inertialize_row); ACLB200_NO_INERTIALIZATION rows are left as
		//             decoded. Phases 4b and 5 then run as for the object mode when parents are given, and store local rows without them.
		//             k_compose_mirror (aclb200_decompress_tracks_mirrored): requests are 12 byte aclb200_mirrored_request records; a request
		//             whose `mirrored` is neither 0 nor 1 is not sought (it writes nothing). Phase 4c mirrors the rows of each request with
		//             mirrored == 1 in place, one thread per partner pair (obj::mirror_row); phases 4b and 5 as in the inertialized mode.
		template<int NORM, bool PER_TRACK, bool STAGED, bool OUT_STAGED, bool DB, uint32_t COMPOSE>
		__global__ void __launch_bounds__(k_threads_per_block)
		transform_decompress_tracks_kernel(const DecodeParams p)
		{
			constexpr bool PAIRED = COMPOSE == k_compose_additive || COMPOSE == k_compose_blend;
			constexpr bool MASKED = COMPOSE == k_compose_layers_masked;
			constexpr bool LAYERED = COMPOSE == k_compose_layers || MASKED;
			constexpr bool INERT = COMPOSE == k_compose_inertialize;
			constexpr bool MIRROR = COMPOSE == k_compose_mirror;
			// MASKED: a layer slot's op carries the layer's mask index above its low k_layer_op_bits
			auto slot_op = [](uint32_t slot) { return MASKED ? slot & k_layer_op_mask : slot; };
			static_assert(COMPOSE == k_compose_local || OUT_STAGED, "the composed decodes work on poses assembled in shared memory");
			using RS = typename std::conditional<DB, ReqStateDB, ReqState>::type;
			// dynamic shared memory: RS[requests_per_block] (LAYERED: then LayerSlot[requests_per_block]) | key frame windows | pose staging
			extern __shared__ __align__(16) uint8_t s_dynamic[];
			__shared__ __align__(8) uint64_t s_barrier;
			RS* s_req = reinterpret_cast<RS*>(s_dynamic);
			uint8_t* s_stage_bytes = s_dynamic + p.smem_stage_offset;
			const uint32_t* s_stage = reinterpret_cast<const uint32_t*>(s_stage_bytes);
			uint8_t* s_out = s_dynamic + p.smem_out_offset;

			const uint32_t first_request = blockIdx.x * p.requests_per_block;
			const uint32_t num_requests = min(p.requests_per_block, p.num_requests - first_request);
			// LAYERED: what each layer does, and the block's stacks (requests_per_block and num_requests are multiples of L; recomputed or
			// read back where they are used rather than kept live through the decode)
			LayerSlot* s_layer = reinterpret_cast<LayerSlot*>(s_dynamic + size_t(p.requests_per_block) * sizeof(RS));
			auto num_stacks = [&]() { return s_layer[0].num_stacks; };
			auto first_stack = [&]() { return blockIdx.x * fast_div(p.requests_per_block, p.magic_layers); };
			if (LAYERED && threadIdx.x == 0)
				s_layer[0].num_stacks = fast_div(num_requests, p.magic_layers);
			InertializationSlot* s_inert = reinterpret_cast<InertializationSlot*>(s_layer);
			MirrorSlot* s_mirror = reinterpret_cast<MirrorSlot*>(s_layer);

			if (STAGED)
			{
				if (threadIdx.x == 0)
					mbar_init(&s_barrier, num_requests);
				__syncthreads();
			}

			// ---- phase 1: seek + stage the two key frames ----
			if (threadIdx.x < num_requests)
			{
				RS rs;
				if constexpr (LAYERED)
				{
					// an OFF layer (or an unknown op) never reaches the clip table; an ADDITIVE layer above the base takes the writer defaults
					const aclb200_layer* stack_layers = reinterpret_cast<const aclb200_layer*>(p.requests) + first_request;
					const uint32_t stack = fast_div(threadIdx.x, p.magic_layers);
					const aclb200_layer layer = stack_layers[threadIdx.x];
					bool base = layer.op == ACLB200_LAYER_BLEND || layer.op == ACLB200_LAYER_ADDITIVE;
					for (uint32_t below = stack * p.num_layers; below < threadIdx.x; ++below)
						base = base && __ldg(&stack_layers[below].op) == ACLB200_LAYER_OFF;
					uint32_t op = layer.op > ACLB200_LAYER_ADDITIVE ? k_layer_unknown : (base ? k_layer_base : layer.op);
					// MASKED: the mask index of a BLEND or ADDITIVE layer above the base, read beside its record
					if (MASKED && p.layer_masks != nullptr && (op == ACLB200_LAYER_BLEND || op == ACLB200_LAYER_ADDITIVE))
					{
						const uint32_t mask = __ldg(p.layer_masks + first_request + threadIdx.x);
						if (mask != ACLB200_LAYER_NO_MASK)
							op = mask < p.num_masks ? op | ((mask + 1) << k_layer_op_bits) : k_layer_unknown;
					}
					s_layer[threadIdx.x].op = op;
					s_layer[threadIdx.x].weight = layer.weight;
					rs.num_tracks = 0;
					if (layer.op == ACLB200_LAYER_BLEND || layer.op == ACLB200_LAYER_ADDITIVE)
						seek_request<DB>(p, layer.pose, first_stack() + stack, rs);
				}
				else if constexpr (INERT)
				{
					// {clip, sample_time, record, elapsed, halflife}, five words at 4 byte alignment
					const uint32_t* words = reinterpret_cast<const uint32_t*>(p.requests) + uint64_t(first_request + threadIdx.x) * 5;
					const uint32_t record = __ldg(words + 2);
					rs.num_tracks = 0;
					if (record == ACLB200_NO_INERTIALIZATION || record < p.num_records)
						seek_request<DB>(p, aclb200_request{ __ldg(words), __uint_as_float(__ldg(words + 1)) }, first_request + threadIdx.x, rs);
					s_inert[threadIdx.x] = InertializationSlot{ record, __uint_as_float(__ldg(words + 3)), __uint_as_float(__ldg(words + 4)), 0u };
				}
				else if constexpr (MIRROR)
				{
					// {clip, sample_time, mirrored}, three words at 4 byte alignment
					const uint32_t* words = reinterpret_cast<const uint32_t*>(p.requests) + uint64_t(first_request + threadIdx.x) * 3;
					const uint32_t mirrored = __ldg(words + 2);
					rs.num_tracks = 0;
					if (mirrored <= 1u)
						seek_request<DB>(p, aclb200_request{ __ldg(words), __uint_as_float(__ldg(words + 1)) }, first_request + threadIdx.x, rs);
					s_mirror[threadIdx.x].mirrored = mirrored;
				}
				else
					seek_transform<DB, RS, PAIRED>(p, first_request + threadIdx.x, rs);
				rs.out = p.out + uint64_t(first_request + threadIdx.x) * p.pose_stride;
				if (STAGED)
				{
					if (rs.num_tracks != 0 && (rs.num_animated[0] | rs.num_animated[1] | rs.num_animated[2]) != 0)
					{
						uint32_t src_byte[2], bytes[2];
#pragma unroll
						for (int k = 0; k < 2; ++k)
						{
							src_byte[k] = (rs.kf_bit[k] >> 3) & ~15u;
							rs.bit_base[k] = rs.kf_bit[k] - src_byte[k] * 8;
							rs.word_base[k] = (threadIdx.x * 2 + k) * (p.stage_bytes >> 2);
							bytes[k] = min((((rs.bit_base[k] + rs.pose_bits[k] + 7) >> 3) + 8 + 15) & ~15u, p.stage_bytes);
						}
						mbar_arrive_expect_tx(&s_barrier, bytes[0] + bytes[1]);
#pragma unroll
						for (int k = 0; k < 2; ++k)
							bulk_copy_g2s(s_stage_bytes + size_t(rs.word_base[k]) * 4, stream_base(rs, k) + src_byte[k], bytes[k], &s_barrier);
					}
					else
						mbar_arrive(&s_barrier);
				}
				s_req[threadIdx.x] = rs;
			}
			__syncthreads();

			// ---- LAYERED: one thread per stack finds its base layer, or that the stack writes nothing (read after phase 4c's barrier) ----
			if constexpr (LAYERED)
			{
				if (threadIdx.x < num_stacks())
				{
					uint32_t base = k_no_base;
					bool valid = true;
					for (uint32_t layer = threadIdx.x * p.num_layers; layer < (threadIdx.x + 1) * p.num_layers; ++layer)
					{
						const uint32_t op = slot_op(s_layer[layer].op);
						if (op == ACLB200_LAYER_OFF)
							continue;
						const uint32_t tracks = s_req[layer].num_tracks;
						if (op == k_layer_unknown || tracks == 0 || (base != k_no_base && tracks != s_req[base].num_tracks))
							valid = false;
						if (base == k_no_base)
							base = layer;
					}
					s_layer[threadIdx.x].stack_base = valid ? base : k_no_base;
				}
			}

			// ---- phase 2: constant and default sub-tracks, one thread per (request, bone) ----
			{
				const uint32_t num_slots = num_requests * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t local_request = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - local_request * p.max_tracks;
					const RS& rs = s_req[local_request];
					if (bone >= rs.num_tracks)
						continue;
					const uint64_t desc = __ldg(reinterpret_cast<const unsigned long long*>(rs.image + rs.bone_table_off) + bone);
					uint8_t* pose = OUT_STAGED ? s_out + size_t(local_request) * p.smem_pose_bytes : rs.out;
					constant_sub_tracks<NORM, false>(p, rs, bone, desc, pose + size_t(bone) * p.bone_stride,
						(COMPOSE == k_compose_additive && (local_request & 1u) != 0) || (LAYERED && slot_op(s_layer[local_request].op) == ACLB200_LAYER_ADDITIVE));
				}
			}

			if (STAGED)
				mbar_wait(&s_barrier, 0);

			// ---- phase 3: animated rotations, one thread per (request, animated rotation sub-track) ----
			if (p.max_animated[0] != 0)
			{
				const uint32_t num_slots = num_requests * p.max_animated[0];
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t local_request = fast_div(slot, p.magic_rot);
					const uint32_t rank = slot - local_request * p.max_animated[0];
					const RS& rs = s_req[local_request];
					if (rs.num_tracks == 0 || rank >= rs.num_animated[0])
						continue;
					float rotation[4];
					const uint32_t bone = animated_rotation<NORM, PER_TRACK, false, STAGED>(p, rs, s_stage, rank, rs.alpha, rotation);
					if (skip_sub_track(p, 0, bone))
						continue;
					uint8_t* pose = OUT_STAGED ? s_out + size_t(local_request) * p.smem_pose_bytes : rs.out;
					write_rotation(p.layout, pose + size_t(bone) * p.bone_stride, rotation);
				}
			}

			// ---- phase 4: animated translations then scales ----
			const uint32_t max_vectors = p.max_animated[1] + p.max_animated[2];
			if (max_vectors != 0)
			{
				const uint32_t num_slots = num_requests * max_vectors;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t local_request = fast_div(slot, p.magic_vec);
					uint32_t rank = slot - local_request * max_vectors;
					const RS& rs = s_req[local_request];
					uint32_t kind = 1;
					if (rank >= p.max_animated[1])
					{
						rank -= p.max_animated[1];
						kind = 2;
					}
					if (rs.num_tracks == 0 || rank >= rs.num_animated[kind])
						continue;
					float value[3];
					const uint32_t bone = animated_vector<PER_TRACK, false, STAGED>(p, rs, s_stage, kind, rank, rs.alpha, value);
					if (skip_sub_track(p, kind, bone))
						continue;
					uint8_t* pose = OUT_STAGED ? s_out + size_t(local_request) * p.smem_pose_bytes : rs.out;
					write_vector(p.layout, pose + size_t(bone) * p.bone_stride, kind, value);
				}
			}

			// ---- phase 4c: one thread per (pair, bone) applies the additive row (request 2r + 1) to the base row (request 2r), in place;
			// a pair whose halves differ in bone count (or name an invalid clip) is left alone and never stored ----
			if constexpr (COMPOSE == k_compose_additive)
			{
				__syncthreads();
				uint32_t flags = 0;
				const uint32_t num_slots = (num_requests >> 1) * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t pair = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - pair * p.max_tracks;
					const RS& base = s_req[2 * pair];
					const uint32_t additive_tracks = s_req[2 * pair + 1].num_tracks;
					if (bone >= base.num_tracks || additive_tracks != base.num_tracks)
						continue;
					uint32_t format = p.additive_format;
					if (p.clip_additive_formats != nullptr)
					{
						format = __ldg(p.clip_additive_formats + s_req[2 * pair + 1].clip);
						format = format <= ACLB200_ADDITIVE_ADDITIVE1 ? format : ACLB200_ADDITIVE_NONE;		// apply_additive_to_base's `default:`
					}
					uint8_t* row = s_out + size_t(2 * pair) * p.smem_pose_bytes + size_t(bone) * p.bone_stride;
					flags |= obj::apply_additive_row(row, row, row + p.smem_pose_bytes, format, p.layout == ACLB200_LAYOUT_QVV40);
				}
				flags = __reduce_or_sync(0xFFFFFFFFu, flags);
				if ((threadIdx.x & 31u) == 0 && flags != 0 && p.object_flags != nullptr)
					atomicOr(p.object_flags, flags);
			}

			// ---- phase 4c, blend: one thread per (pair, bone) lerps the from row (request 2r) towards the to row (request 2r + 1), in place,
			// with the pair's weight; pairs whose halves differ in bone count are left alone as above ----
			if constexpr (COMPOSE == k_compose_blend)
			{
				__syncthreads();
				const uint32_t first_pair = first_request >> 1;
				const uint32_t num_slots = (num_requests >> 1) * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t pair = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - pair * p.max_tracks;
					const uint32_t from_tracks = s_req[2 * pair].num_tracks;
					if (bone >= from_tracks || s_req[2 * pair + 1].num_tracks != from_tracks)
						continue;
					const float weight = p.blend_weights != nullptr ? __ldg(p.blend_weights + first_pair + pair) : p.blend_weight;
					uint8_t* row = s_out + size_t(2 * pair) * p.smem_pose_bytes + size_t(bone) * p.bone_stride;
					obj::blend_row(row, row, row + p.smem_pose_bytes, weight, p.layout == ACLB200_LAYOUT_QVV40);
				}
			}

			// ---- phase 4c, layers: one thread per (stack, bone) folds the layers above the base into the base row, in place and in layer order:
			// BLEND lerps towards the layer's row, ADDITIVE applies the layer's row to the running one, OFF is passed over; stacks that write
			// nothing are left alone. MASKED scales a masked layer's weight per bone and weighs ADDITIVE layers ----
			if constexpr (LAYERED)
			{
				__syncthreads();
				const uint32_t num_slots = num_stacks() * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t stack = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - stack * p.max_tracks;
					const uint32_t base = s_layer[stack].stack_base;
					if (base == k_no_base || bone >= s_req[base].num_tracks)
						continue;
					uint8_t* row = s_out + size_t(base) * p.smem_pose_bytes + size_t(bone) * p.bone_stride;
					for (uint32_t layer = base + 1; layer < (stack + 1) * p.num_layers; ++layer)
					{
						const uint32_t slot = s_layer[layer].op;
						const uint32_t op = slot_op(slot);
						float weight = s_layer[layer].weight;
						if (MASKED && slot > k_layer_op_mask)
						{
							// the layer's weight at this bone is weight * mask[bone]; a mask of +-0 leaves the running row as it is
							const float mask = __ldg(p.bone_masks + ((slot >> k_layer_op_bits) - 1) * p.mask_stride + bone);
							if (mask == 0.0f)
								continue;
							weight = __fmul_rn(weight, mask);
						}
						uint8_t* layer_row = s_out + size_t(layer) * p.smem_pose_bytes + size_t(bone) * p.bone_stride;
						if (op == ACLB200_LAYER_BLEND)
							obj::blend_row(row, row, layer_row, weight, p.layout == ACLB200_LAYOUT_QVV40);
						else if (op == ACLB200_LAYER_ADDITIVE)
						{
							uint32_t format = p.additive_format;
							if (p.clip_additive_formats != nullptr)
							{
								format = __ldg(p.clip_additive_formats + s_req[layer].clip);
								format = format <= ACLB200_ADDITIVE_ADDITIVE1 ? format : ACLB200_ADDITIVE_NONE;		// apply_additive_to_base's `default:`
							}
							// MASKED, weight != 1: the layer's row becomes qvv_lerp(writer defaults, layer, weight) in place (no other thread
							// reads it), which scales the additive delta of every format
							if (MASKED && weight != 1.0f)
							{
								const bool qvv40 = p.layout == ACLB200_LAYOUT_QVV40;
								const float* defaults = k_writer_default_rows[qvv40][(s_req[layer].clip_flags & k_clip_default_scale_one) != 0];
								obj::blend_row(layer_row, reinterpret_cast<const uint8_t*>(defaults), layer_row, weight, qvv40);
							}
							// (a flag is rare: reported where it is met, so that no accumulator stays live through the fold)
							const uint32_t flags = obj::apply_additive_row(row, row, layer_row, format, p.layout == ACLB200_LAYOUT_QVV40);
							if (flags != 0 && p.object_flags != nullptr)
								atomicOr(p.object_flags, flags);
						}
					}
				}
			}

			// ---- phase 4c, inertialize: one thread per (request, bone) decays the request's record entry onto the row, in place ----
			if constexpr (INERT)
			{
				__syncthreads();
				const uint32_t num_slots = num_requests * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t local_request = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - local_request * p.max_tracks;
					const InertializationSlot inertialization = s_inert[local_request];
					if (bone >= s_req[local_request].num_tracks || inertialization.record == ACLB200_NO_INERTIALIZATION)
						continue;
					uint8_t* row = s_out + size_t(local_request) * p.smem_pose_bytes + size_t(bone) * p.bone_stride;
					const float4* entry = reinterpret_cast<const float4*>(p.records + uint64_t(inertialization.record) * p.record_stride
						+ uint64_t(bone) * ACLB200_INERTIALIZATION_ENTRY_BYTES);
					obj::inertialize_row(row, row, entry, obj::inertialization_decay(inertialization.elapsed, inertialization.halflife),
						p.layout == ACLB200_LAYOUT_QVV40);
				}
			}

			// ---- phase 4c, mirror: one thread per (request, bone) of the mirrored requests; the thread of the lower row of each partner pair
			// mirrors both rows in place, so no other thread touches them. The clip's table is indexed like its parents ----
			if constexpr (MIRROR)
			{
				__syncthreads();
				uint32_t flags = 0;
				const uint32_t num_slots = num_requests * p.max_tracks;
				for (uint32_t slot = threadIdx.x; slot < num_slots; slot += k_threads_per_block)
				{
					const uint32_t local_request = fast_div(slot, p.magic_tracks);
					const uint32_t bone = slot - local_request * p.max_tracks;
					const uint32_t num_tracks = s_req[local_request].num_tracks;
					if (bone >= num_tracks || s_mirror[local_request].mirrored != 1u)
						continue;
					const uint32_t skeleton = p.skeleton_offsets != nullptr ? __ldg(p.skeleton_offsets + s_req[local_request].clip) : 0u;
					const aclb200_mirror_entry* table = p.mirror_table + skeleton;
					bool invalid = false;
					const uint32_t partner = obj::mirror_partner(table, bone, num_tracks, invalid);
					if (invalid)
						flags |= ACLB200_ERROR_FLAG_INVALID_MIRROR;
					if (partner < bone)
						continue;
					uint8_t* pose = s_out + size_t(local_request) * p.smem_pose_bytes;
					uint8_t* row = pose + size_t(bone) * p.bone_stride;
					uint8_t* partner_row = pose + size_t(partner) * p.bone_stride;
					obj::mirror_row(row, partner_row, row, partner_row, table + bone, table + partner, p.mirror_axis, p.layout == ACLB200_LAYOUT_QVV40);
				}
				if (flags != 0 && p.object_flags != nullptr)
					atomicOr(p.object_flags, flags);
			}

			// ---- phase 4b: one warp per staged pose walks the clip's skeleton and overwrites the local rows with object rows (PAIRED: the
			// combined row of each pair, when parents are given) ----
			if constexpr (COMPOSE != k_compose_local)
			{
				if ((!PAIRED && !LAYERED && !INERT && !MIRROR) || p.parent_indices != nullptr)
				{
					__syncthreads();
					uint32_t flags = 0;
					constexpr uint32_t step = PAIRED ? 2u : 1u;
					const uint32_t num_items = LAYERED ? num_stacks() : num_requests;
					for (uint32_t item = (threadIdx.x >> 5) * step; item < num_items; item += (k_threads_per_block / 32) * step)
					{
						uint32_t local_request = item;
						if constexpr (LAYERED)
						{
							local_request = s_layer[item].stack_base;
							if (local_request == k_no_base)
								continue;
						}
						const RS& rs = s_req[local_request];
						if (rs.num_tracks == 0 || (PAIRED && s_req[local_request + 1].num_tracks != rs.num_tracks))
							continue;
						const uint32_t skeleton = p.skeleton_offsets != nullptr ? __ldg(p.skeleton_offsets + rs.clip) : 0u;
						uint8_t* pose = s_out + size_t(local_request) * p.smem_pose_bytes;
						flags |= obj::pose_rows_to_object_space(pose, rs.num_tracks, p.parent_indices + skeleton, p.object_kind != ACLB200_OBJECT_QVVF);
						if (p.object_kind == k_object_skinning)
							obj::skin_pose_rows(pose, rs.num_tracks, p.inverse_bind + size_t(skeleton) * 12);
					}
					flags = __reduce_or_sync(0xFFFFFFFFu, flags);
					if ((threadIdx.x & 31u) == 0 && flags != 0 && p.object_flags != nullptr)
						atomicOr(p.object_flags, flags);
				}
			}

			// ---- phase 5: the assembled poses leave shared memory as full, coalesced 16 byte (or 8 byte) stores (PAIRED: row 2r of each
			// pair whose halves match, as output r) ----
			if (OUT_STAGED)
			{
				__syncthreads();
				const uint32_t chunks_per_pose = p.smem_pose_bytes >> 4;
				const uint32_t num_poses = PAIRED ? num_requests >> 1 : (LAYERED ? num_stacks() : num_requests);
				const uint32_t first_pose = PAIRED ? first_request >> 1 : (LAYERED ? first_stack() : first_request);
				const uint32_t num_chunks = num_poses * chunks_per_pose;
				for (uint32_t slot = threadIdx.x; slot < num_chunks; slot += k_threads_per_block)
				{
					const uint32_t local_pose = fast_div(slot, p.magic_chunks);
					uint32_t local_request = PAIRED ? local_pose * 2 : local_pose;
					if constexpr (LAYERED)
					{
						local_request = s_layer[local_pose].stack_base;
						if (local_request == k_no_base)
							continue;
					}
					const uint32_t byte = (slot - local_pose * chunks_per_pose) << 4;
					uint32_t row_bytes = s_req[local_request].num_tracks * p.bone_stride;
					if (PAIRED && s_req[local_request + 1].num_tracks != s_req[local_request].num_tracks)
						row_bytes = 0;
					if (byte >= row_bytes)
						continue;
					const uint8_t* src = s_out + size_t(local_request) * p.smem_pose_bytes + byte;
					uint8_t* dst = p.out + uint64_t(first_pose + local_pose) * p.pose_stride + byte;
					if (p.out_vector16 && byte + 16 <= row_bytes)
						*reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
					else
					{
						*reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
						if (byte + 8 < row_bytes)
							*reinterpret_cast<uint2*>(dst + 8) = *reinterpret_cast<const uint2*>(src + 8);
					}
				}
			}
		}

		// decompress_track_v0, decompression.transform.h:1753-2050: one thread per request, one bone each
		template<int NORM, bool PER_TRACK, bool DB = false>
		__global__ void __launch_bounds__(128)
		transform_decompress_track_kernel(const DecodeParams p)
		{
			const uint32_t request = blockIdx.x * blockDim.x + threadIdx.x;
			if (request >= p.num_requests)
				return;
			typename std::conditional<DB, ReqStateDB, ReqState>::type rs;
			seek_transform<DB>(p, request, rs);
			const uint32_t bone = p.track_indices[request];
			if (bone >= rs.num_tracks)
				return;		// :1766-1768: invalid track index, nothing is written
			uint8_t* out_bone = p.out + uint64_t(request) * p.bone_stride;
			const uint64_t desc = __ldg(reinterpret_cast<const unsigned long long*>(rs.image + rs.bone_table_off) + bone);
			constant_sub_tracks<NORM, true>(p, rs, bone, desc, out_bone);

			if ((uint32_t(desc) & 3) == 2 && !skip_sub_track(p, 0, bone))
			{
				float rotation[4];
				animated_rotation<NORM, PER_TRACK, true, false>(p, rs, nullptr, (uint32_t(desc) >> 2) & k_bone_index_mask, rs.alpha, rotation);
				write_rotation(p.layout, out_bone, rotation);
			}
#pragma unroll
			for (uint32_t kind = 1; kind <= 2; ++kind)
			{
				const uint32_t bits = uint32_t(desc >> (k_bone_kind_shift * kind));
				if ((bits & 3) == 2 && (kind == 1 || (rs.clip_flags & k_clip_has_scale)) && !skip_sub_track(p, kind, bone))
				{
					float value[3];
					animated_vector<PER_TRACK, true, false>(p, rs, nullptr, kind, (bits >> 2) & k_bone_index_mask, rs.alpha, value);
					write_vector(p.layout, out_bone, kind, value);
				}
			}
		}

		__global__ void __launch_bounds__(128)
		transform_debug_seek_kernel(const DecodeParams p, aclb200_seek_state* __restrict__ out)
		{
			const uint32_t request = blockIdx.x * blockDim.x + threadIdx.x;
			if (request >= p.num_requests)
				return;
			ReqState rs;
			seek_transform(p, request, rs);
			aclb200_seek_state st = {};
			st.sample_time = rs.sample_time;
			if (rs.num_tracks != 0)
			{
				st.interpolation_alpha = rs.alpha;
				st.uses_single_segment = rs.single_segment;
				st.looping_policy = rs.looping_policy;
				for (int k = 0; k < 2; ++k)
				{
					st.key_frame_bit_offsets[k] = rs.kf_bit[k];
					st.segment_indices[k] = rs.segment_index[k];
					st.animated_offsets[k] = rs.blob_animated_off[k];
					st.format_offsets[k] = rs.blob_format_off[k];
					st.range_offsets[k] = rs.blob_range_off[k];
				}
			}
			out[request] = st;
		}

		__global__ void __launch_bounds__(128)
		transform_debug_unpack_kernel(const DecodeParams p, uint32_t* __restrict__ out)
		{
			__shared__ ReqState s_req;
			const uint32_t request = blockIdx.x;
			if (threadIdx.x == 0)
				seek_transform(p, request, s_req);
			__syncthreads();
			const ReqState& rs = s_req;
			if (rs.num_tracks == 0)
				return;
			const int k = int(p.debug_which);
			const uint32_t total = rs.num_animated[0] + rs.num_animated[1] + rs.num_animated[2];
			for (uint32_t slot = threadIdx.x; slot < total && slot < p.debug_max_sub_tracks; slot += blockDim.x)
			{
				const Entry e = load_entry(rs, k, slot);
				const bool four = slot < rs.num_animated[0] && (rs.clip_flags & k_clip_rot_full);
				uint32_t xi, yi, zi, wi;
				unpack_sample_ints<false>(rs, nullptr, k, e, four, xi, yi, zi, wi);
				uint32_t* dst = out + (size_t(request) * p.debug_max_sub_tracks + slot) * 4;
				dst[0] = xi; dst[1] = yi; dst[2] = zi;
				dst[3] = e.offset_code & 0xFFu;
			}
		}

		// ---------------------------------------------------------------------------------------------------
		// scalar tracks: seek_v0 + decompress_tracks_v0 / decompress_track_v0, decompression/impl/decompression.scalar.h:181-705
		// ---------------------------------------------------------------------------------------------------
		struct ScalarReqState
		{
			const uint8_t* image;
			const ScalarTrackDesc* tracks;
			uint8_t* out;
			float    alpha;
			uint32_t num_tracks;
			uint32_t kf_bit[2];
			uint32_t constant_off;
			uint32_t range_off;
			uint32_t stream_off;
		};

		__device__ void seek_scalar(const DecodeParams& p, uint32_t request_index, ScalarReqState& rs)
		{
			rs.num_tracks = 0;
			const aclb200_request request = p.requests[request_index];
			if (request.clip >= p.num_clips)
				return;
			const ClipDesc& clip = p.clips[request.clip];
			if (clip.num_tracks == 0 || clip.num_samples == 0)
				return;

			uint32_t rounding_policy, requested_looping, looping_policy;
			float duration;
			request_policies(p, request_index, rounding_policy, requested_looping);
			resolve_looping(p, clip, requested_looping, looping_policy, duration);
			float sample_time = request.sample_time;
			if (p.clamp_sample_time)
				sample_time = fminf(fmaxf(sample_time, 0.0f), duration);

			uint32_t key_frame0, key_frame1;
			float alpha;
			find_key_frames(clip.num_samples, clip.sample_rate, sample_time, rounding_policy, looping_policy, key_frame0, key_frame1, alpha);

			rs.image = p.data + clip.data_offset;
			rs.tracks = reinterpret_cast<const ScalarTrackDesc*>(rs.image + clip.bone_table_offset);
			rs.alpha = alpha;
			rs.num_tracks = clip.num_tracks;
			rs.kf_bit[0] = key_frame0 * clip.num_animated_total;		// num_bits_per_frame, decompression.scalar.h:208-209
			rs.kf_bit[1] = key_frame1 * clip.num_animated_total;
			rs.constant_off = clip.const_rot_offset;
			rs.range_off = clip.const_vec_offset;
			rs.stream_off = clip.seg_table_offset;
		}

		__device__ __forceinline__ uint32_t read_stream32(const uint32_t* words, uint32_t bit)
		{
			const uint32_t hi = __ldg(words + (bit >> 5));
			const uint32_t lo = __ldg(words + (bit >> 5) + 1);
			return __funnelshift_l(lo, hi, bit & 31);
		}

		template<int COMPONENTS, bool PER_TRACK>
		__device__ __forceinline__ void decode_scalar_track(const DecodeParams& p, const ScalarReqState& rs, uint32_t track, float* out)
		{
			const uint4 raw = __ldg(reinterpret_cast<const uint4*>(rs.tracks) + track);
			const uint32_t num_bits = raw.y & 0xFFu;
			const uint32_t value_index = raw.y >> 8;
			const float inv_max = __uint_as_float(raw.z);
			float alpha = rs.alpha;
			if (PER_TRACK)
				alpha = apply_rounding_policy(rs.alpha, track_rounding_policy(p, track));	// decompression.scalar.h:235-247,273-280

			if (num_bits == 0)
			{
				const float* constants = reinterpret_cast<const float*>(rs.image + rs.constant_off) + value_index;
#pragma unroll
				for (int c = 0; c < COMPONENTS; ++c)
					out[c] = __ldg(constants + c);
				return;
			}

			const uint32_t* words = reinterpret_cast<const uint32_t*>(rs.image + rs.stream_off);
			const uint32_t bit0 = rs.kf_bit[0] + raw.x;
			const uint32_t bit1 = rs.kf_bit[1] + raw.x;
			if (num_bits == 32)
			{
#pragma unroll
				for (int c = 0; c < COMPONENTS; ++c)
				{
					const float v0 = __uint_as_float(read_stream32(words, bit0 + 32 * c));
					const float v1 = __uint_as_float(read_stream32(words, bit1 + 32 * c));
					out[c] = lerp(v0, v1, alpha);
				}
				return;
			}

			const float* range = reinterpret_cast<const float*>(rs.image + rs.range_off) + value_index;
#pragma unroll
			for (int c = 0; c < COMPONENTS; ++c)
			{
				const uint32_t i0 = read_stream32(words, bit0 + num_bits * c) >> (32 - num_bits);
				const uint32_t i1 = read_stream32(words, bit1 + num_bits * c) >> (32 - num_bits);
				const float range_min = __ldg(range + c);
				const float range_extent = __ldg(range + COMPONENTS + c);
				const float v0 = fmuladd(fmul(u2f(i0), inv_max), range_extent, range_min);
				const float v1 = fmuladd(fmul(u2f(i1), inv_max), range_extent, range_min);
				out[c] = lerp(v0, v1, alpha);
			}
		}

		// ---------------------------------------------------------------------------------------------------
		// scalar decompress_tracks, chained: a block takes a batch of consecutive requests. Warp 0 runs the seek (one lane per request)
		// and groups the requests that play one clip forward (request i + 1 starts on the key frame request i ends on): a group's key
		// frames are ONE contiguous piece of the clip's bit stream, staged in shared memory by one TMA copy. Then one thread per
		// (group, track): the track's descriptor and range are loaded once per group, every key frame value is unpacked once
		// (n + 1 unpacks for n requests instead of 2 n), and each request's sample leaves with a coalesced store (consecutive threads
		// hold consecutive tracks). Groups whose window does not fit the pool read the stream from global memory instead.
		// ---------------------------------------------------------------------------------------------------
		constexpr uint32_t k_scalar_threads = 256;
		constexpr uint32_t k_scalar_max_batch = 32;

		struct alignas(16) ScalarHot
		{
			const uint8_t* image;
			uint8_t* out;
			float    alpha;					// (alpha, bit1) are read together, once per request and thread
			uint32_t bit1;					// key frame bit addresses: inside the pool (staged) or inside the clip's stream
			uint32_t bit0;
			uint32_t num_tracks;			// 0 => invalid request
			uint32_t tracks_off, constant_off, range_off, stream_off;
			uint32_t group;					// (first request) | (count << 8) | (staged << 16), valid on the group's first request
			uint32_t track_range_off;
		};
		static_assert(sizeof(ScalarHot) == 64, "ScalarHot is 64 bytes");

		template<int COMPONENTS>
		__device__ __forceinline__ void scalar_key_frame_value(const uint32_t* pool_words, const uint32_t* stream_words, bool staged, uint32_t bit, uint32_t num_bits,
			float inv_max, const float range_min[COMPONENTS], const float range_extent[COMPONENTS], float value[COMPONENTS])
		{
			const uint32_t* words = staged ? pool_words : stream_words;
#pragma unroll
			for (int c = 0; c < COMPONENTS; ++c)
			{
				const uint32_t at = bit + (num_bits == 32 ? 32u : num_bits) * c;
				const uint32_t hi = staged ? words[at >> 5] : __ldg(words + (at >> 5));
				const uint32_t lo = staged ? words[(at >> 5) + 1] : __ldg(words + (at >> 5) + 1);
				const uint32_t raw = __funnelshift_l(lo, hi, at & 31);
				if (num_bits == 32)
					value[c] = __uint_as_float(raw);
				else
					value[c] = fmuladd(fmul(u2f(raw >> (32 - num_bits)), inv_max), range_extent[c], range_min[c]);		// decompression.scalar.h:317-346
			}
		}

		template<int COMPONENTS, bool PER_TRACK>
		__global__ void __launch_bounds__(k_scalar_threads)
		scalar_tracks_pipeline_kernel(const DecodeParams p)
		{
			extern __shared__ __align__(16) uint8_t s_dynamic[];		// the key frame pool
			__shared__ ScalarHot s_hot[k_scalar_max_batch];
			__shared__ __align__(8) uint64_t s_barrier;
			__shared__ uint32_t s_num_groups;
			__shared__ uint32_t s_group_first[k_scalar_max_batch];

			const uint32_t first_request = blockIdx.x * p.requests_per_block;
			const uint32_t num_requests = min(p.requests_per_block, p.num_requests - first_request);
			const uint32_t pool_bytes = p.smem_bytes;
			if (threadIdx.x == 0)
				mbar_init(&s_barrier, 32);
			__syncthreads();

			if (threadIdx.x < 32)
			{
				// ---- seek + grouping + window staging, one lane per request ----
				const uint32_t lane = threadIdx.x;
				const bool active = lane < num_requests;
				ScalarReqState rs;
				rs.num_tracks = 0;
				uint32_t clip_index = 0xFFFFFFFFu, bits_per_frame = 0;
				if (active)
				{
					seek_scalar(p, first_request + lane, rs);
					if (rs.num_tracks != 0)
					{
						clip_index = p.requests[first_request + lane].clip;
						bits_per_frame = p.clips[clip_index].num_animated_total;
					}
				}
				const bool valid = rs.num_tracks != 0;
				const uint32_t kf0 = valid ? rs.kf_bit[0] : 0u, kf1 = valid ? rs.kf_bit[1] : 0u;
				const bool mergeable = valid && kf1 >= kf0 && bits_per_frame != 0;
				const uint32_t prev_clip = __shfl_up_sync(0xFFFFFFFFu, mergeable ? clip_index : 0xFFFFFFFFu, 1);
				const uint32_t prev_kf1 = __shfl_up_sync(0xFFFFFFFFu, kf1, 1);
				const bool join = lane > 0 && mergeable && clip_index == prev_clip && kf0 == prev_kf1;
				const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane);
				const uint32_t heads = __ballot_sync(0xFFFFFFFFu, !join);
				const uint32_t group_start = 31 - __clz(heads & lanes_le);
				const uint32_t heads_after = lane == 31 ? 0u : (heads & (0xFFFFFFFEu << lane));
				const uint32_t group_end = heads_after != 0 ? uint32_t(__ffs(heads_after) - 1) : 32u;
				const bool head = !join;
				const uint32_t head_kf0 = __shfl_sync(0xFFFFFFFFu, kf0, group_start);
				const uint32_t last_kf1 = __shfl_sync(0xFFFFFFFFu, kf1, (group_end - 1) & 31);

				// the group's window: 16 byte aligned start, every key frame from the first request's first to the last request's second,
				// 16 bytes of tail for the last value's second word
				const uint32_t src_byte = (head_kf0 >> 3) & ~15u;
				uint32_t window_bytes = 0;
				if (head && mergeable)
					window_bytes = ((((last_kf1 + bits_per_frame - src_byte * 8) + 7) >> 3) + 16 + 15) & ~15u;
				// pool offsets: exclusive prefix sum of the heads' window sizes
				uint32_t offset = window_bytes;
#pragma unroll
				for (uint32_t d = 1; d < 32; d <<= 1)
				{
					const uint32_t below = __shfl_up_sync(0xFFFFFFFFu, offset, d);
					if (lane >= d)
						offset += below;
				}
				offset -= window_bytes;
				const bool staged_head = head && mergeable && window_bytes != 0 && offset + window_bytes <= pool_bytes;
				const bool staged = __shfl_sync(0xFFFFFFFFu, staged_head, group_start);
				const uint32_t window_offset = __shfl_sync(0xFFFFFFFFu, offset, group_start);

				if (active)
				{
					ScalarHot h;
					h.image = rs.image;
					h.out = p.out + uint64_t(first_request + lane) * p.pose_stride;
					h.alpha = rs.alpha;
					h.num_tracks = rs.num_tracks;
					h.tracks_off = valid ? uint32_t(reinterpret_cast<const uint8_t*>(rs.tracks) - rs.image) : 0u;
					h.constant_off = rs.constant_off;
					h.range_off = rs.range_off;
					h.stream_off = rs.stream_off;
					h.bit0 = staged ? window_offset * 8 + (kf0 - src_byte * 8) : kf0;
					h.bit1 = staged ? window_offset * 8 + (kf1 - src_byte * 8) : kf1;
					h.group = lane | ((group_end - group_start) << 8) | (staged ? 1u << 16 : 0u);
					h.track_range_off = clip_index != 0xFFFFFFFFu ? p.clips[clip_index].track_range_offset : 0u;
					s_hot[lane] = h;
				}
				if (head && active)
					s_group_first[__popc(heads & lanes_le) - 1] = lane;
				if (lane == 0)
					s_num_groups = __popc(heads & (num_requests >= 32 ? 0xFFFFFFFFu : ((1u << num_requests) - 1u)));
				if (staged_head && active)
				{
					mbar_arrive_expect_tx(&s_barrier, window_bytes);
					bulk_copy_g2s(s_dynamic + offset, rs.image + rs.stream_off + src_byte, window_bytes, &s_barrier);
				}
				else
					mbar_arrive(&s_barrier);
			}
			__syncthreads();
			mbar_wait(&s_barrier, 0);

			// ---- group by group, one thread per track ----
			// The chain: request r interpolates (value at its first key frame, value at its second); its second key frame is the next
			// request's first, so each request costs ONE unpack. Requests go two at a time: the two new key frame values travel as one
			// f32x2 pair through the range expansion and the interpolation (exact: see muladd2 in device_common.cuh). Constant tracks
			// ride along (their range is (constant, 0)) and a final select keeps the constant itself, as the reference writes it
			// (decompression.scalar.h:289-315): no divergence between the lanes of a warp.
			const uint32_t* pool_words = reinterpret_cast<const uint32_t*>(s_dynamic);
			const uint64_t pose_stride = p.pose_stride;
			const uint32_t num_groups = s_num_groups;
			for (uint32_t group = 0; group < num_groups; ++group)
			{
				const uint32_t first = s_group_first[group];
				const ScalarHot& h0 = s_hot[first];
				const uint32_t num_tracks = h0.num_tracks;
				if (num_tracks == 0)
					continue;
				const uint32_t count = (h0.group >> 8) & 0xFFu;
				const bool staged = (h0.group >> 16) != 0;
				const uint4* descs = reinterpret_cast<const uint4*>(h0.image + h0.tracks_off);		// ScalarTrackDesc
				const float* ranges = reinterpret_cast<const float*>(h0.image + h0.track_range_off);
				const uint32_t* stream_words = reinterpret_cast<const uint32_t*>(h0.image + h0.stream_off);
				const uint32_t first_bit = h0.bit0;
				uint8_t* group_out = h0.out;
				const uint32_t hot_addr = smem_u32(&s_hot[first].alpha);

				auto tracks_loop = [&](auto staged_tag)
				{
					constexpr bool STAGED = decltype(staged_tag)::value;
					const uint32_t* words = STAGED ? pool_words : stream_words;
					auto word = [&](uint32_t index) { return STAGED ? words[index] : __ldg(words + index); };
					auto store = [&](uint8_t* row, int c, float v) { asm volatile("st.global.f32 [%0], %1;" :: "l"(row + c * 4), "f"(v) : "memory"); };
					auto load_track = [&](uint32_t track, uint4& desc, float range_min[COMPONENTS], float range_extent[COMPONENTS])
					{
						desc = make_uint4(0, 1, 0, 0);
						if (track >= num_tracks)
							return;
						desc = __ldg(descs + track);
#pragma unroll
						for (int c = 0; c < COMPONENTS; ++c)
						{
							range_min[c] = __ldg(ranges + size_t(track) * COMPONENTS * 2 + c);
							range_extent[c] = __ldg(ranges + size_t(track) * COMPONENTS * 2 + COMPONENTS + c);
						}
					};
					// the next track's descriptor and range are requested while the current track is being decoded
					uint4 next_desc;
					float next_min[COMPONENTS], next_extent[COMPONENTS];
					load_track(threadIdx.x, next_desc, next_min, next_extent);
					for (uint32_t track = threadIdx.x; track < num_tracks; track += k_scalar_threads)
					{
						const uint4 desc = next_desc;
						float range_min[COMPONENTS], range_extent[COMPONENTS];
#pragma unroll
						for (int c = 0; c < COMPONENTS; ++c)
						{
							range_min[c] = next_min[c];
							range_extent[c] = next_extent[c];
						}
						load_track(track + k_scalar_threads, next_desc, next_min, next_extent);

						const uint32_t stored_bits = desc.y & 0xFFu;
						const bool constant = stored_bits == 0;
						const float inv_max = __uint_as_float(desc.z);
						const uint32_t policy = PER_TRACK ? track_rounding_policy(p, track) : ACLB200_ROUND_NONE;
						uint8_t* out = group_out + size_t(track) * COMPONENTS * 4;
						if (stored_bits == 32)
						{
							// raw 32 bit samples: no range, plain interpolation (rare: the compressor keeps them for tracks it cannot quantise)
							float start[COMPONENTS];
							scalar_key_frame_value<COMPONENTS>(pool_words, stream_words, STAGED, first_bit + desc.x, 32, inv_max, range_min, range_extent, start);
							for (uint32_t r = 0; r < count; ++r)
							{
								uint2 h;
								asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(h.x), "=r"(h.y) : "r"(hot_addr + r * uint32_t(sizeof(ScalarHot))));
								float end[COMPONENTS];
								scalar_key_frame_value<COMPONENTS>(pool_words, stream_words, STAGED, h.y + desc.x, 32, inv_max, range_min, range_extent, end);
								const float alpha = PER_TRACK ? apply_rounding_policy(__uint_as_float(h.x), policy) : __uint_as_float(h.x);
#pragma unroll
								for (int c = 0; c < COMPONENTS; ++c)
								{
									store(out + uint64_t(r) * pose_stride, c, lerp(start[c], end[c], alpha));
									start[c] = end[c];
								}
							}
							continue;
						}

						const uint32_t num_bits = constant ? 1u : stored_bits;		// constant tracks: any defined shift, the value is replaced below
						const uint32_t down = 32 - num_bits;
						auto unpack = [&](uint32_t at) { return __funnelshift_l(word((at >> 5) + 1), word(at >> 5), at & 31) >> down; };
						float start[COMPONENTS];
#pragma unroll
						for (int c = 0; c < COMPONENTS; ++c)
							start[c] = fmuladd(fmul(u2f(unpack(first_bit + desc.x + num_bits * c)), inv_max), range_extent[c], range_min[c]);		// decompression.scalar.h:317-346
						uint32_t r = 0;
						for (; r + 2 <= count; r += 2)
						{
							uint2 ha, hb;		// (alpha, bit1) of requests r and r + 1
							asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(ha.x), "=r"(ha.y) : "r"(hot_addr + r * uint32_t(sizeof(ScalarHot))));
							asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(hb.x), "=r"(hb.y) : "r"(hot_addr + (r + 1) * uint32_t(sizeof(ScalarHot))));
							float alpha_a = __uint_as_float(ha.x), alpha_b = __uint_as_float(hb.x);
							if (PER_TRACK)
							{
								alpha_a = apply_rounding_policy(alpha_a, policy);		// decompression.scalar.h:235-247,273-280
								alpha_b = apply_rounding_policy(alpha_b, policy);
							}
							const float2 alpha = make_float2(alpha_a, alpha_b);
							uint8_t* row_a = out + uint64_t(r) * pose_stride;
							uint8_t* row_b = row_a + pose_stride;
#pragma unroll
							for (int c = 0; c < COMPONENTS; ++c)
							{
								float2 end = mul2(make_float2(u2f(unpack(ha.y + desc.x + num_bits * c)), u2f(unpack(hb.y + desc.x + num_bits * c))), inv_max);
								end = muladd2(end, range_extent[c], range_min[c]);
								const float2 begin = make_float2(start[c], end.x);
								// rtm::scalar_lerp / vector_lerp: end * alpha + (start - start * alpha)
								const float2 value = add2(mul2(end, alpha), sub2(begin, mul2(begin, alpha)));
								store(row_a, c, constant ? range_min[c] : value.x);
								store(row_b, c, constant ? range_min[c] : value.y);
								start[c] = end.y;
							}
						}
						if (r < count)
						{
							uint2 h;
							asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(h.x), "=r"(h.y) : "r"(hot_addr + r * uint32_t(sizeof(ScalarHot))));
							const float alpha = PER_TRACK ? apply_rounding_policy(__uint_as_float(h.x), policy) : __uint_as_float(h.x);
#pragma unroll
							for (int c = 0; c < COMPONENTS; ++c)
							{
								const float end = fmuladd(fmul(u2f(unpack(h.y + desc.x + num_bits * c)), inv_max), range_extent[c], range_min[c]);
								store(out + uint64_t(r) * pose_stride, c, constant ? range_min[c] : lerp(start[c], end, alpha));
							}
						}
					}
				};
				if (staged)
					tracks_loop(std::true_type());
				else
					tracks_loop(std::false_type());
			}
		}

		template<int COMPONENTS, bool PER_TRACK>
		__global__ void __launch_bounds__(128)
		scalar_decompress_track_kernel(const DecodeParams p)
		{
			const uint32_t request = blockIdx.x * blockDim.x + threadIdx.x;
			if (request >= p.num_requests)
				return;
			ScalarReqState rs;
			seek_scalar(p, request, rs);
			const uint32_t track = p.track_indices[request];
			if (track >= rs.num_tracks)
				return;
			float value[COMPONENTS];
			decode_scalar_track<COMPONENTS, PER_TRACK>(p, rs, track, value);
			float* dst = reinterpret_cast<float*>(p.out) + size_t(request) * COMPONENTS;
#pragma unroll
			for (int c = 0; c < COMPONENTS; ++c)
				dst[c] = value[c];
		}

		uint32_t division_magic(uint32_t divisor)
		{
			// floor(v / d) == mulhi(v, magic) for v < 2^32 / d, which every slot index here satisfies (v < 2^18 + 2048 items, d <= 2^18)
			return divisor <= 1 ? 0u : uint32_t((uint64_t(1) << 32) / divisor) + 1u;
		}

		using DecodeKernel = void (*)(DecodeParams);

		// The transform_decompress_tracks_kernel instance of a launch, nullptr for a choice no plan makes: a composed decode always assembles
		// its poses in shared memory. configure_kernels walks every choice through here, so every kernel a launch can pick is configured.
		DecodeKernel tracks_kernel(uint32_t normalization, bool per_track, bool database, bool staged, bool out_staged, uint32_t compose)
		{
			return with_constant<3>(normalization, [&](auto NORM) { return with_bool(per_track, [&](auto PER_TRACK) {
				return with_bool(database, [&](auto DB) { return with_bool(staged, [&](auto STAGED) { return with_bool(out_staged, [&](auto OUT_STAGED) {
					return with_constant<k_compose_count>(compose, [&](auto COMPOSE) -> DecodeKernel {
						if constexpr (COMPOSE != k_compose_local && !OUT_STAGED)
							return nullptr;
						else
							return transform_decompress_tracks_kernel<NORM, PER_TRACK, STAGED, OUT_STAGED, DB, COMPOSE>;
					}); }); }); }); }); });
		}

		DecodeKernel track_kernel(uint32_t normalization, bool per_track, bool database)
		{
			return with_constant<3>(normalization, [&](auto NORM) { return with_bool(per_track, [&](auto PER_TRACK) {
				return with_bool(database, [&](auto DB) -> DecodeKernel { return transform_decompress_track_kernel<NORM, PER_TRACK, DB>; }); }); });
		}

		// aclb200_apply_additive_to_base: one thread per (pose, bone) of QVV48 rows; out may be either input (a thread reads its two rows
		// before it writes its own)
		__global__ void __launch_bounds__(256)
		apply_additive_kernel(const uint8_t* base_poses, const uint8_t* additive_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
			uint64_t pose_stride, uint32_t additive_format, uint32_t* out_flags)
		{
			uint32_t flags = 0;
			const uint64_t num_items = num_poses * num_tracks;
			for (uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; item < num_items; item += uint64_t(gridDim.x) * blockDim.x)
			{
				const uint64_t pose = item / num_tracks;
				const uint64_t offset = pose * pose_stride + (item - pose * num_tracks) * 48;
				flags |= obj::apply_additive_row(out + offset, base_poses + offset, additive_poses + offset, additive_format, false);
			}
			flags = __reduce_or_sync(0xFFFFFFFFu, flags);
			if ((threadIdx.x & 31u) == 0 && flags != 0 && out_flags != nullptr)
				atomicOr(out_flags, flags);
		}

		// aclb200_blend_poses: one thread per (pose, bone) of QVV48 rows; out may be either input (a thread reads its two rows before it
		// writes its own)
		__global__ void __launch_bounds__(256)
		blend_poses_kernel(const uint8_t* from_poses, const uint8_t* to_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
			uint64_t pose_stride, float weight, const float* weights)
		{
			const uint64_t num_items = num_poses * num_tracks;
			for (uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; item < num_items; item += uint64_t(gridDim.x) * blockDim.x)
			{
				const uint64_t pose = item / num_tracks;
				const uint64_t offset = pose * pose_stride + (item - pose * num_tracks) * 48;
				obj::blend_row(out + offset, from_poses + offset, to_poses + offset, weights != nullptr ? __ldg(weights + pose) : weight, false);
			}
		}

		// aclb200_local_to_skinning: one warp per pose. The warp stages the pose's local rows in its share of shared memory with coalesced 16
		// byte loads, runs the walk and the skinning step the skinning decodes run (so the two routes are bit-identical by construction) and
		// stores the rows the same way. out may be the input: a warp has read its whole pose before it writes any of it.
		__global__ void __launch_bounds__(256)
		local_to_skinning_kernel(const uint8_t* local_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride,
			const uint32_t* parents, const float* inverse_bind, uint32_t* out_flags)
		{
			extern __shared__ __align__(16) uint8_t s_poses[];
			const uint32_t lane = threadIdx.x & 31u;
			const uint32_t warps_per_block = blockDim.x >> 5;
			const uint32_t chunks = num_tracks * 3;		// 16 byte chunks per pose
			uint4* staged = reinterpret_cast<uint4*>(s_poses) + size_t(threadIdx.x >> 5) * chunks;
			uint32_t flags = 0;
			for (uint64_t pose = uint64_t(blockIdx.x) * warps_per_block + (threadIdx.x >> 5); pose < num_poses; pose += uint64_t(gridDim.x) * warps_per_block)
			{
				const uint4* src = reinterpret_cast<const uint4*>(local_poses + pose * pose_stride);
				for (uint32_t chunk = lane; chunk < chunks; chunk += 32)
					staged[chunk] = src[chunk];
				__syncwarp();
				flags |= obj::pose_rows_to_object_space(reinterpret_cast<uint8_t*>(staged), num_tracks, parents, true);
				obj::skin_pose_rows(reinterpret_cast<uint8_t*>(staged), num_tracks, inverse_bind);
				__syncwarp();
				uint4* dst = reinterpret_cast<uint4*>(out + pose * pose_stride);
				for (uint32_t chunk = lane; chunk < chunks; chunk += 32)
					dst[chunk] = staged[chunk];
				__syncwarp();
			}
			flags = __reduce_or_sync(0xFFFFFFFFu, flags);
			if (lane == 0 && flags != 0 && out_flags != nullptr)
				atomicOr(out_flags, flags);
		}
	}

	uint32_t pose_operation_blocks(uint64_t num_poses, uint32_t num_tracks, int num_sms)
	{
		const uint64_t blocks_needed = (num_poses * num_tracks + 255) / 256;
		return uint32_t(blocks_needed < uint64_t(num_sms) * 16 ? blocks_needed : uint64_t(num_sms) * 16);
	}

	// Called once per context: lets the staged kernels use large dynamic shared memory windows. `max_dynamic_smem` comes in as the
	// device's opt-in limit and goes out as what a launch may actually request.
	cudaError_t configure_kernels(int& max_dynamic_smem)
	{
		const int optin_limit = max_dynamic_smem - 1024;
		int available = optin_limit;
		cudaError_t error = cudaSuccess;
		for (uint32_t choice = 0; choice < 3 * 16 * k_compose_count && error == cudaSuccess; ++choice)
		{
			// (normalization, per_track | database << 1 | staged << 2 | out_staged << 3, compose)
			const uint32_t compose = choice % k_compose_count, bits = choice / k_compose_count % 16, normalization = choice / (16 * k_compose_count);
			const DecodeKernel kernel = tracks_kernel(normalization, bits & 1, bits & 2, bits & 4, bits & 8, compose);
			if (kernel == nullptr)
				continue;
			// the opt-in limit covers static + dynamic shared memory
			cudaFuncAttributes attributes;
			error = cudaFuncGetAttributes(&attributes, kernel);
			if (error != cudaSuccess)
				break;
			const int kernel_available = optin_limit - int(attributes.sharedSizeBytes);
			if (kernel_available < available)
				available = kernel_available;
			error = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kernel_available);
		}
		if (error == cudaSuccess) error = cudaFuncSetAttribute(local_to_skinning_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin_limit);
		if (error == cudaSuccess) error = configure_pipeline_kernels(optin_limit, available);
		if (error == cudaSuccess) error = configure_error_kernels(available);
		max_dynamic_smem = available;
		return error;
	}

	// requests_per_block, the division magics and the shared memory carve-up of a launch
	// compose != local: the composed decodes need every pose in shared memory, so a pose that does not fit gives up key frame staging
	// instead (params.smem_bytes then tells the caller whether one request fits at all)
	// additive, blend: requests_per_block stays even, so that the two halves of a pair always share a block; layers: a multiple of
	// params.num_layers, so that a stack never spans two blocks (and each request carries a LayerSlot beside its state)
	void plan_launch(DecodeParams& params, uint32_t max_key_frame_bytes, int max_dynamic_smem, bool allow_output_staging, bool database,
		uint32_t compose)
	{
		const bool force_output_staging = compose != k_compose_local;
		const bool pairs = compose == k_compose_additive || compose == k_compose_blend;
		const bool layers = compose == k_compose_layers || compose == k_compose_layers_masked;
		// a LayerSlot, an InertializationSlot or a MirrorSlot beside each request state
		const bool slots = layers || compose == k_compose_inertialize || compose == k_compose_mirror;
		const uint32_t state_bytes = (database ? uint32_t(sizeof(ReqStateDB)) : uint32_t(sizeof(ReqState))) + (slots ? uint32_t(sizeof(LayerSlot)) : 0u);
		const uint32_t max_tracks = params.max_tracks == 0 ? 1 : params.max_tracks;
		const uint32_t budget = uint32_t(max_dynamic_smem > 0 ? max_dynamic_smem : 0);
		// ~28 KB of shared memory per block keeps 8 blocks resident per SM
		const uint32_t block_budget = budget < 28u * 1024u ? budget : 28u * 1024u;

		// bytes per staged key frame: alignment skew + the key frame + the extra word the funnel shift reads, 16 byte granular
		uint32_t stage_bytes = max_key_frame_bytes != 0 ? ((max_key_frame_bytes + 48 + 15) & ~15u) : 0u;
		uint32_t pose_bytes = allow_output_staging || force_output_staging ? ((max_tracks * params.bone_stride + 15) & ~15u) : 0u;

		uint32_t requests_per_block = k_target_items_per_block / max_tracks;
		if (requests_per_block < 1) requests_per_block = 1;
		if (requests_per_block > k_max_requests_per_block) requests_per_block = k_max_requests_per_block;
		const uint32_t step = layers ? params.num_layers : (pairs ? 2u : 1u);
		requests_per_block = requests_per_block < step ? step : requests_per_block - requests_per_block % step;

		auto bytes_needed = [&](uint32_t requests) { return requests * (state_bytes + 2 * stage_bytes + pose_bytes); };
		while (requests_per_block > step && bytes_needed(requests_per_block) > block_budget)
			requests_per_block -= step;
		// a single request that does not fit: give up output staging first, then key frame staging
		if (bytes_needed(requests_per_block) > budget && !force_output_staging)
			pose_bytes = 0;
		if (bytes_needed(requests_per_block) > budget)
			stage_bytes = 0;

		params.requests_per_block = requests_per_block;
		params.stage_bytes = stage_bytes;
		params.smem_pose_bytes = pose_bytes;
		params.smem_stage_offset = (requests_per_block * state_bytes + 15) & ~15u;
		params.smem_out_offset = params.smem_stage_offset + requests_per_block * 2 * stage_bytes;
		params.smem_bytes = params.smem_out_offset + requests_per_block * pose_bytes;
		params.magic_tracks = division_magic(max_tracks);
		params.magic_rot = division_magic(params.max_animated[0]);
		params.magic_vec = division_magic(params.max_animated[1] + params.max_animated[2]);
		params.magic_chunks = division_magic(pose_bytes >> 4);
		params.magic_layers = division_magic(params.num_layers);
		params.out_vector16 = ((uint64_t(reinterpret_cast<uintptr_t>(params.out)) | params.pose_stride) & 15) == 0 ? 1u : 0u;
	}

	// Both math modes run these exact kernels (only the pipeline kernel has a fast variant)
	cudaError_t launch_transform_decompress_tracks(const DecodeParams& params, uint32_t compose, bool database, cudaStream_t stream)
	{
		const DecodeKernel kernel = tracks_kernel(params.normalization, params.per_track_rounding != 0, database, params.stage_bytes != 0,
			params.smem_pose_bytes != 0, compose);
		if (kernel == nullptr)
			return cudaErrorInvalidConfiguration;
		const uint32_t blocks = (params.num_requests + params.requests_per_block - 1) / params.requests_per_block;
		kernel<<<blocks, k_threads_per_block, params.smem_bytes, stream>>>(params);
		return cudaGetLastError();
	}

	cudaError_t launch_transform_decompress_track(const DecodeParams& params, bool database, cudaStream_t stream)
	{
		const uint32_t blocks = (params.num_requests + 127) / 128;
		track_kernel(params.normalization, params.per_track_rounding != 0, database)<<<blocks, 128, 0, stream>>>(params);
		return cudaGetLastError();
	}

	cudaError_t launch_apply_additive(const uint8_t* base_poses, const uint8_t* additive_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
		uint64_t pose_stride, uint32_t additive_format, uint32_t* flags, int num_sms, cudaStream_t stream)
	{
		apply_additive_kernel<<<pose_operation_blocks(num_poses, num_tracks, num_sms), 256, 0, stream>>>(base_poses, additive_poses, out, num_poses,
			num_tracks, pose_stride, additive_format, flags);
		return cudaGetLastError();
	}

	cudaError_t launch_blend_poses(const uint8_t* from_poses, const uint8_t* to_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks,
		uint64_t pose_stride, float weight, const float* weights, int num_sms, cudaStream_t stream)
	{
		blend_poses_kernel<<<pose_operation_blocks(num_poses, num_tracks, num_sms), 256, 0, stream>>>(from_poses, to_poses, out, num_poses, num_tracks,
			pose_stride, weight, weights);
		return cudaGetLastError();
	}

	// up to 8 warps per block, as many as whole poses fit the block's shared memory
	uint32_t local_to_skinning_warps(uint32_t num_tracks, int max_dynamic_smem)
	{
		const uint64_t fit = uint64_t(max_dynamic_smem > 0 ? max_dynamic_smem : 0) / (uint64_t(num_tracks) * 48);
		return uint32_t(fit < 8 ? fit : 8);
	}

	cudaError_t launch_local_to_skinning(const uint8_t* local_poses, uint8_t* out, uint64_t num_poses, uint32_t num_tracks, uint64_t pose_stride,
		const uint32_t* parents, const float* inverse_bind, uint32_t* flags, uint32_t warps, int num_sms, cudaStream_t stream)
	{
		const uint64_t blocks_needed = (num_poses + warps - 1) / warps;
		const uint32_t blocks = uint32_t(blocks_needed < uint64_t(num_sms) * 16 ? blocks_needed : uint64_t(num_sms) * 16);
		local_to_skinning_kernel<<<blocks, warps * 32, size_t(warps) * num_tracks * 48, stream>>>(local_poses, out, num_poses, num_tracks, pose_stride,
			parents, inverse_bind, flags);
		return cudaGetLastError();
	}

	cudaError_t launch_transform_debug_seek(const DecodeParams& params, aclb200_seek_state* d_out, cudaStream_t stream)
	{
		const uint32_t blocks = (params.num_requests + 127) / 128;
		transform_debug_seek_kernel<<<blocks, 128, 0, stream>>>(params, d_out);
		return cudaGetLastError();
	}

	cudaError_t launch_transform_debug_unpack(const DecodeParams& params, uint32_t* d_out, cudaStream_t stream)
	{
		transform_debug_unpack_kernel<<<params.num_requests, 128, 0, stream>>>(params, d_out);
		return cudaGetLastError();
	}

	// The key frame pool of the chained scalar kernel: 4 blocks of 48 KB + statics stay resident per SM
#ifndef ACLB200_SCALAR_POOL_KB
#define ACLB200_SCALAR_POOL_KB 48
#endif
	constexpr uint32_t k_scalar_pool_bytes = ACLB200_SCALAR_POOL_KB * 1024u;

	template<int COMPONENTS, bool PER_TRACK>
	static cudaError_t launch_scalar_pipeline(const DecodeParams& params, cudaStream_t stream)
	{
		static bool configured = false;		// (idempotent; a race only repeats the call)
		if (!configured)
		{
			const cudaError_t error = cudaFuncSetAttribute(scalar_tracks_pipeline_kernel<COMPONENTS, PER_TRACK>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(k_scalar_pool_bytes));
			if (error != cudaSuccess)
				return error;
			configured = true;
		}
		const uint32_t blocks = (params.num_requests + params.requests_per_block - 1) / params.requests_per_block;
		scalar_tracks_pipeline_kernel<COMPONENTS, PER_TRACK><<<blocks, k_scalar_threads, params.smem_bytes, stream>>>(params);
		return cudaGetLastError();
	}

	template<bool PER_TRACK>
	static cudaError_t launch_scalar_tracks(const DecodeParams& params, uint32_t components, cudaStream_t stream)
	{
		switch (components)
		{
		case 1: return launch_scalar_pipeline<1, PER_TRACK>(params, stream);
		case 2: return launch_scalar_pipeline<2, PER_TRACK>(params, stream);
		case 3: return launch_scalar_pipeline<3, PER_TRACK>(params, stream);
		default: return launch_scalar_pipeline<4, PER_TRACK>(params, stream);
		}
	}

	// requests per block and the key frame pool of a scalar decompress_tracks launch: as many requests as chained key frames fit the pool
	void plan_scalar_launch(DecodeParams& params, uint32_t max_key_frame_bytes)
	{
		const uint32_t frame_bytes = max_key_frame_bytes + 48;
		uint32_t requests_per_block = frame_bytes != 0 ? k_scalar_pool_bytes / frame_bytes : 1;
		if (requests_per_block > 1) --requests_per_block;		// n chained requests read n + 1 key frames
		if (requests_per_block < 1) requests_per_block = 1;
		if (requests_per_block > k_scalar_max_batch) requests_per_block = k_scalar_max_batch;
		// small clips: keep a block busy with at least ~4096 (request, track) items when the pool allows
		params.requests_per_block = requests_per_block;
		params.smem_bytes = k_scalar_pool_bytes;
		params.magic_tracks = division_magic(params.max_tracks == 0 ? 1 : params.max_tracks);
	}

	template<bool PER_TRACK>
	static cudaError_t launch_scalar_track(const DecodeParams& params, uint32_t components, cudaStream_t stream)
	{
		const uint32_t blocks = (params.num_requests + 127) / 128;
		switch (components)
		{
		case 1: scalar_decompress_track_kernel<1, PER_TRACK><<<blocks, 128, 0, stream>>>(params); break;
		case 2: scalar_decompress_track_kernel<2, PER_TRACK><<<blocks, 128, 0, stream>>>(params); break;
		case 3: scalar_decompress_track_kernel<3, PER_TRACK><<<blocks, 128, 0, stream>>>(params); break;
		default: scalar_decompress_track_kernel<4, PER_TRACK><<<blocks, 128, 0, stream>>>(params); break;
		}
		return cudaGetLastError();
	}

	cudaError_t launch_scalar_decompress_tracks(const DecodeParams& params, cudaStream_t stream)
	{
		const uint32_t components = params.bone_stride / 4;
		return params.per_track_rounding ? launch_scalar_tracks<true>(params, components, stream) : launch_scalar_tracks<false>(params, components, stream);
	}

	cudaError_t launch_scalar_decompress_track(const DecodeParams& params, cudaStream_t stream)
	{
		const uint32_t components = params.bone_stride / 4;
		return params.per_track_rounding ? launch_scalar_track<true>(params, components, stream) : launch_scalar_track<false>(params, components, stream);
	}
}
