// acl_b200/csrc/device_common.cuh -- device-side building blocks shared by the kernels: exact float helpers, TMA / mbarrier
// wrappers, the fused seek, the bit stream readers and the per sub-track decoders. See kernels.cu for the arithmetic contract.
#pragma once

#include "context.h"

#include <type_traits>

namespace aclb200
{
	namespace dev
	{
		constexpr uint32_t k_threads_per_block = 256;
		constexpr uint32_t k_max_requests_per_block = 64;
		constexpr uint32_t k_target_items_per_block = 512;

		// The kernel instance of a launch from its run-time choices: f(std::integral_constant<uint32_t, value>) for a run-time value < N,
		// f(std::bool_constant<value>) for a run-time bool; f returns the instance
		template<uint32_t N, typename F>
		auto with_constant(uint32_t value, F f)
		{
			if constexpr (N == 1)
				return f(std::integral_constant<uint32_t, 0>());
			else
				return value == N - 1 ? f(std::integral_constant<uint32_t, N - 1>()) : with_constant<N - 1>(value, f);
		}

		template<typename F>
		auto with_bool(bool value, F f)
		{
			return value ? f(std::true_type()) : f(std::false_type());
		}

		// ---------------------------------------------------------------------------------------------------
		// exact float helpers
		// ---------------------------------------------------------------------------------------------------
		__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
		__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
		__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
		// rtm::vector_mul_add(a, b, c) == (a * b) + c, two roundings
		__device__ __forceinline__ float fmuladd(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }
		// rtm::vector_neg_mul_sub(a, b, c) == c - (a * b)
		__device__ __forceinline__ float fnegmulsub(float a, float b, float c) { return __fsub_rn(c, __fmul_rn(a, b)); }
		__device__ __forceinline__ float u2f(uint32_t v) { return __uint2float_rn(v); }

		// ---- f32x2 pair arithmetic ----
		// The x and y lanes of a pair run the same operation sequence. sm_90 has no packed f32x2 pipe, so each helper issues one scalar
		// IEEE operation per lane; __fmul_rn / __fadd_rn / __fsub_rn are never contracted into an FMA, which keeps every result
		// bit-identical to the reference's separate mul and add.
		__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(fmul(a.x, b.x), fmul(a.y, b.y)); }
		__device__ __forceinline__ float2 mul2(float2 a, float b) { return make_float2(fmul(a.x, b), fmul(a.y, b)); }
		__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(fadd(a.x, b.x), fadd(a.y, b.y)); }		// a + b
		__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(fsub(a.x, b.x), fsub(a.y, b.y)); }		// a - b
		__device__ __forceinline__ float2 muladd2(float2 a, float2 b, float2 c) { return make_float2(fmuladd(a.x, b.x, c.x), fmuladd(a.y, b.y, c.y)); }
		__device__ __forceinline__ float2 muladd2(float2 a, float b, float c) { return make_float2(fmuladd(a.x, b, c), fmuladd(a.y, b, c)); }
		__device__ __forceinline__ float2 negmulsub2(float2 a, float2 b, float2 c) { return make_float2(fnegmulsub(a.x, b.x, c.x), fnegmulsub(a.y, b.y, c.y)); }

		// ---------------------------------------------------------------------------------------------------
		// TMA bulk copy + mbarrier (PTX ISA: cp.async.bulk, mbarrier)
		// ---------------------------------------------------------------------------------------------------
		__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

		__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
		{
			asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
			asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		}

		__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
		{
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
		}

		__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
		{
			asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
		}

		__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
		{
			uint32_t done;
			do
			{
				asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
					: "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
			} while (!done);
		}

		// 1-D bulk tensor-less TMA copy global -> shared (SASS: UBLKCP); dst, src and bytes are multiples of 16
		__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
		{
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
				:: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
		}

		// ---------------------------------------------------------------------------------------------------
		// per request state, written by one thread, read by every item thread of the request
		// ---------------------------------------------------------------------------------------------------
		struct alignas(16) ReqState
		{
			const uint8_t* image;
			uint8_t* out;
			float    alpha;
			uint32_t num_tracks;			// 0 => nothing to decode (invalid request or empty clip)
			uint32_t clip_flags;
			uint32_t single_segment;
			uint32_t entries_off[2];		// image relative Entry tables of the two key frames' segments
			uint32_t stream_off[2];			// image relative streams
			uint32_t bit_base[2];			// staged: bit of the key frame inside its shared memory window; else key_frame_bit_offsets
			uint32_t word_base[2];			// staged: first word of the window inside the block's staging area
			uint32_t anim_off;
			uint32_t bone_table_off;
			uint32_t const_rot_off;
			uint32_t const_vec_off;
			uint32_t num_animated[3];
			uint32_t num_constant_trans;
			// extras reported by the seek parity hook
			float    sample_time;
			uint32_t kf_bit[2];
			uint32_t segment_index[2];
			uint32_t blob_format_off[2];
			uint32_t blob_range_off[2];
			uint32_t blob_animated_off[2];
			uint32_t pose_bits[2];
			uint32_t looping_policy;
			uint32_t clip;
		};

		// The request state of the database kernels (seek_transform<true>): a key frame streamed in from a database tier lies outside
		// the clip image, so each key frame carries its own stream base.
		struct ReqStateDB : ReqState
		{
			const uint8_t* stream[2];		// 16 byte aligned: byte-swapped words, key frame k starts at bit kf_bit[k] of stream[k]
		};

		__device__ __forceinline__ const uint8_t* stream_base(const ReqState& rs, int k) { return rs.image + rs.stream_off[k]; }
		__device__ __forceinline__ const uint8_t* stream_base(const ReqStateDB& rs, int k) { return rs.stream[k]; }

		// Where key frame `key_frame` (segment relative) of one segment lives: the clip, or a database tier whose metadata
		// ((samples_offset << 32) | sample_indices, database_runtime_segment_header) holds it (decompression.transform.h:329-352,483-505)
		__device__ __forceinline__ void locate_tier_key_frame(const DecodeParams& p, uint64_t medium, uint64_t low, uint32_t key_frame,
			uint32_t& sample_indices, const uint8_t*& tier_data, uint32_t& tier_offset)
		{
			const uint64_t bit = uint64_t(1) << (31 - key_frame);
			if ((medium & bit) != 0)
			{
				sample_indices = uint32_t(medium);
				tier_data = p.db_bulk[0];
				tier_offset = uint32_t(medium >> 32);
			}
			else if ((low & bit) != 0)
			{
				sample_indices = uint32_t(low);
				tier_data = p.db_bulk[1];
				tier_offset = uint32_t(low >> 32);
			}
		}

		// apply_rounding_policy, core/impl/interpolation_utils.impl.h:261-278
		__device__ __forceinline__ float apply_rounding_policy(float alpha, uint32_t policy)
		{
			if (policy == ACLB200_ROUND_FLOOR) return 0.0f;
			if (policy == ACLB200_ROUND_CEIL) return 1.0f;
			if (policy == ACLB200_ROUND_NEAREST) return floorf(fadd(alpha, 0.5f));
			return alpha;
		}

		// find_linear_interpolation_alpha, core/impl/interpolation_utils.impl.h:224-253 with rounding_policy == none
		__device__ __forceinline__ float interpolation_alpha_none(float sample_index, uint32_t index0, uint32_t index1)
		{
			if (index0 == index1)
				return 0.0f;
			if (index0 < index1)
				return __fdiv_rn(fsub(sample_index, u2f(index0)), u2f(index1 - index0));
			return fsub(sample_index, u2f(index0));
		}

		// Looping policy + clamp duration: initialize_v0 / set_looping_policy_v0, decompression.transform.h:120-129,186-204
		__device__ __forceinline__ void resolve_looping(const DecodeParams& p, const ClipDesc& clip, uint32_t requested, uint32_t& policy, float& duration)
		{
			if (!p.wrapping)
				policy = ACLB200_LOOP_CLAMP;
			else if (requested == ACLB200_LOOP_AS_COMPRESSED)
				policy = (clip.flags & k_clip_wrap) ? ACLB200_LOOP_WRAP : ACLB200_LOOP_CLAMP;
			else
				policy = requested;
			duration = policy == ACLB200_LOOP_WRAP ? clip.duration_wrap : clip.duration_clamp;
		}

		// seek(sample_time, rounding_policy) and set_looping_policy(policy) of one request: the batch wide options, or the request's
		// own pair (aclb200_options::d_request_policies)
		__device__ __forceinline__ void request_policies(const DecodeParams& p, uint32_t request_index, uint32_t& rounding, uint32_t& looping)
		{
			rounding = p.rounding_policy;
			looping = p.looping_policy;
			if (p.request_policies != nullptr)
			{
				const uint32_t pair = __ldg(reinterpret_cast<const unsigned short*>(p.request_policies) + request_index);
				rounding = (pair & 0xFFu) <= ACLB200_ROUND_NEAREST ? (pair & 0xFFu) : ACLB200_ROUND_NONE;
				looping = (pair >> 8) <= ACLB200_LOOP_AS_COMPRESSED ? (pair >> 8) : ACLB200_LOOP_AS_COMPRESSED;
			}
		}

		// track_writer::skip_all_*() || skip_track_*(track), core/track_writer.h:181-191 (kind 0 rotation, 1 translation, 2 scale)
		__device__ __forceinline__ bool skip_sub_track(const DecodeParams& p, uint32_t kind, uint32_t track)
		{
			uint32_t bits = p.skip_all;
			if (p.skip_tracks != nullptr)
				bits |= __ldg(p.skip_tracks + track);
			return ((bits >> kind) & 1u) != 0;
		}

		// find_linear_interpolation_samples_with_sample_rate, core/impl/interpolation_utils.impl.h:143-201
		__device__ __forceinline__ void find_key_frames(uint32_t num_samples, float sample_rate, float sample_time, uint32_t rounding_policy,
			uint32_t looping_policy, uint32_t& key_frame0, uint32_t& key_frame1, float& alpha)
		{
			const uint32_t last_sample_index = num_samples - 1;
			float sample_index = fmul(sample_time, sample_rate);
			uint32_t sample_index0 = __float2uint_rz(sample_index);
			const uint32_t next_sample_index = sample_index0 + 1;
			uint32_t sample_index1;
			if (looping_policy == ACLB200_LOOP_CLAMP)
				sample_index1 = min(next_sample_index, last_sample_index);
			else if (sample_index0 > last_sample_index)
			{
				sample_index = 0.0f;
				sample_index0 = 0;
				sample_index1 = 0;
			}
			else
				sample_index1 = next_sample_index >= num_samples ? 0 : next_sample_index;
			key_frame0 = sample_index0;
			key_frame1 = sample_index1;
			alpha = apply_rounding_policy(fsub(sample_index, u2f(sample_index0)), rounding_policy);
		}

		// seek_v0 for transform clips, decompression.transform.h:206-563. DB == false: no database bound (a clip bound to one decodes
		// from its resident key frames, as a context initialised without the database does). DB == true: the tier branches with the
		// clip set's bound database (RS = ReqStateDB). `policy_index` picks the request's entry of p.request_policies (the composed decodes
		// share one entry between the requests of an output).
		template<bool DB = false, class RS = ReqState>
		__device__ __forceinline__ void seek_request(const DecodeParams& p, const aclb200_request request, uint32_t policy_index, RS& rs)
		{
			rs.num_tracks = 0;
			rs.sample_time = -1.0f;
			if (request.clip >= p.num_clips)
				return;
			const ClipDesc& clip = p.clips[request.clip];
			if (clip.num_tracks == 0)
				return;

			const uint8_t* image = p.data + clip.data_offset;

			uint32_t rounding_policy, requested_looping, looping_policy;
			float duration;
			request_policies(p, policy_index, rounding_policy, requested_looping);
			resolve_looping(p, clip, requested_looping, looping_policy, duration);

			float sample_time = request.sample_time;
			if (p.clamp_sample_time)
				sample_time = fminf(fmaxf(sample_time, 0.0f), duration);		// rtm::scalar_clamp, :215-216

			uint32_t key_frame0, key_frame1;
			float alpha;
			find_key_frames(clip.num_samples, clip.sample_rate, sample_time, rounding_policy, looping_policy, key_frame0, key_frame1, alpha);

			const SegDesc* segs = reinterpret_cast<const SegDesc*>(image + clip.seg_table_offset);
			const bool stripped = (clip.flags & k_clip_stripped) != 0;
			uint32_t segment_index0 = 0, segment_index1 = 0;
			uint32_t segment_key_frame0, segment_key_frame1;
			// DB: the clip's first database segment (0xFFFFFFFF: not bound) and the tier buffer + byte offset of each key frame
			// that lives in a tier (tier_data == nullptr: it lives in the clip, :548-556)
			const uint32_t db_segment = DB ? __ldg(p.db_first_segment + request.clip) : 0xFFFFFFFFu;
			const uint8_t* tier_data0 = nullptr;
			const uint8_t* tier_data1 = nullptr;
			uint32_t tier_offset0 = 0, tier_offset1 = 0;

			if (clip.num_segments == 1)
			{
				if (stripped)
				{
					// :272-362
					uint32_t sample_indices = segs[0].sample_indices;
					const float sample_index = fadd(alpha, u2f(key_frame0));
					uint64_t medium = 0, low = 0;
					if (DB && db_segment != 0xFFFFFFFFu)
					{
						medium = __ldg(p.db_tiers + 2 * size_t(db_segment));
						low = __ldg(p.db_tiers + 2 * size_t(db_segment) + 1);
						sample_indices |= uint32_t(medium) | uint32_t(low);
					}
					const uint32_t candidates0 = sample_indices & (0xFFFFFFFFu << (31 - key_frame0));
					key_frame0 = 31 - (__ffs(candidates0) - 1);						// count_trailing_zeros
					const uint32_t candidates1 = sample_indices & (0xFFFFFFFFu >> key_frame1);
					key_frame1 = __clz(candidates1);
					alpha = interpolation_alpha_none(sample_index, key_frame0, key_frame1);
					uint32_t sample_indices0 = segs[0].sample_indices, sample_indices1 = sample_indices0;
					if (DB)
					{
						locate_tier_key_frame(p, medium, low, key_frame0, sample_indices0, tier_data0, tier_offset0);
						locate_tier_key_frame(p, medium, low, key_frame1, sample_indices1, tier_data1, tier_offset1);
					}
					segment_key_frame0 = __popc(~(0xFFFFFFFFu >> key_frame0) & sample_indices0);
					segment_key_frame1 = __popc(~(0xFFFFFFFFu >> key_frame1) & sample_indices1);
				}
				else
				{
					segment_key_frame0 = key_frame0;
					segment_key_frame1 = key_frame1;
				}
			}
			else
			{
				// :372-409, segment_start_indices ends with a 0xFFFFFFFF sentinel (compression/impl/write_segment_data.h:48-65)
				const uint32_t* start_indices = reinterpret_cast<const uint32_t*>(image + clip.start_indices_offset);
				const uint32_t approx_segment_index = key_frame0 / clip.samples_per_segment;
				const uint32_t start_segment_index = approx_segment_index > 0 ? approx_segment_index - 1 : 0;
				for (uint32_t i = 0; i < 4; ++i)
				{
					const uint32_t segment_index = start_segment_index + i;
					const uint32_t start = start_indices[segment_index];
					if (key_frame0 < start)
					{
						segment_index0 = segment_index - 1;
						if (p.wrapping && key_frame1 == 0)
							segment_index1 = 0;
						else
							segment_index1 = key_frame1 < start ? segment_index0 : segment_index;
						break;
					}
				}
				const uint32_t start0 = start_indices[segment_index0];
				const uint32_t start1 = start_indices[segment_index1];
				segment_key_frame0 = key_frame0 - start0;
				segment_key_frame1 = key_frame1 - start1;

				if (stripped)
				{
					// :411-515
					uint32_t sample_indices0 = segs[segment_index0].sample_indices;
					uint32_t sample_indices1 = segs[segment_index1].sample_indices;
					const float sample_index = fadd(alpha, u2f(key_frame0));
					uint64_t medium0 = 0, low0 = 0, medium1 = 0, low1 = 0;
					if (DB && db_segment != 0xFFFFFFFFu)
					{
						medium0 = __ldg(p.db_tiers + 2 * size_t(db_segment + segment_index0));
						low0 = __ldg(p.db_tiers + 2 * size_t(db_segment + segment_index0) + 1);
						sample_indices0 |= uint32_t(medium0) | uint32_t(low0);
						medium1 = __ldg(p.db_tiers + 2 * size_t(db_segment + segment_index1));
						low1 = __ldg(p.db_tiers + 2 * size_t(db_segment + segment_index1) + 1);
						sample_indices1 |= uint32_t(medium1) | uint32_t(low1);
					}
					const uint32_t candidates0 = sample_indices0 & (0xFFFFFFFFu << (31 - segment_key_frame0));
					segment_key_frame0 = 31 - (__ffs(candidates0) - 1);
					const uint32_t candidates1 = sample_indices1 & (0xFFFFFFFFu >> segment_key_frame1);
					segment_key_frame1 = __clz(candidates1);
					alpha = interpolation_alpha_none(sample_index, start0 + segment_key_frame0, start1 + segment_key_frame1);
					if (DB)
					{
						sample_indices0 = segs[segment_index0].sample_indices;
						sample_indices1 = segs[segment_index1].sample_indices;
						locate_tier_key_frame(p, medium0, low0, segment_key_frame0, sample_indices0, tier_data0, tier_offset0);
						locate_tier_key_frame(p, medium1, low1, segment_key_frame1, sample_indices1, tier_data1, tier_offset1);
					}
					segment_key_frame0 = __popc(~(0xFFFFFFFFu >> segment_key_frame0) & sample_indices0);
					segment_key_frame1 = __popc(~(0xFFFFFFFFu >> segment_key_frame1) & sample_indices1);
				}
			}

			const SegDesc seg0 = segs[segment_index0];
			const SegDesc seg1 = segs[segment_index1];

			rs.image = image;
			rs.clip = request.clip;
			rs.alpha = alpha;
			rs.num_tracks = clip.num_tracks;
			rs.clip_flags = clip.flags;
			rs.single_segment = segment_index0 == segment_index1;
			rs.kf_bit[0] = segment_key_frame0 * seg0.pose_bit_size;				// :558-559
			rs.kf_bit[1] = segment_key_frame1 * seg1.pose_bit_size;
			rs.bit_base[0] = rs.kf_bit[0];
			rs.bit_base[1] = rs.kf_bit[1];
			rs.word_base[0] = rs.word_base[1] = 0;
			rs.stream_off[0] = seg0.stream_offset;
			rs.stream_off[1] = seg1.stream_offset;
			rs.entries_off[0] = seg0.entries_offset;
			rs.entries_off[1] = seg1.entries_offset;
			rs.pose_bits[0] = seg0.pose_bit_size;
			rs.pose_bits[1] = seg1.pose_bit_size;
			rs.anim_off = clip.anim_table_offset;
			rs.bone_table_off = clip.bone_table_offset;
			rs.const_rot_off = clip.const_rot_offset;
			rs.const_vec_off = clip.const_vec_offset;
			rs.num_constant_trans = clip.num_constant[1];
			for (int k = 0; k < 3; ++k)
				rs.num_animated[k] = clip.num_animated[k];
			rs.sample_time = sample_time;
			rs.segment_index[0] = segment_index0;
			rs.segment_index[1] = segment_index1;
			rs.blob_format_off[0] = seg0.blob_format_offset;
			rs.blob_format_off[1] = seg1.blob_format_offset;
			rs.blob_range_off[0] = seg0.blob_range_offset;
			rs.blob_range_off[1] = seg1.blob_range_offset;
			rs.blob_animated_off[0] = seg0.blob_animated_offset;
			rs.blob_animated_off[1] = seg1.blob_animated_offset;
			rs.looping_policy = looping_policy;
			if constexpr (DB)
			{
				// the tier buffers hold byte-swapped words from offset 0 (database.cpp): the key frame starts at bit
				// 8 * samples_offset + segment_key_frame * animated_pose_bit_size, read from the 16 byte aligned word below it
				rs.stream[0] = image + seg0.stream_offset;
				rs.stream[1] = image + seg1.stream_offset;
				if (tier_data0 != nullptr)
				{
					rs.stream[0] = tier_data0 + (tier_offset0 & ~15u);
					rs.kf_bit[0] += (tier_offset0 & 15u) * 8;
					rs.bit_base[0] = rs.kf_bit[0];
				}
				if (tier_data1 != nullptr)
				{
					rs.stream[1] = tier_data1 + (tier_offset1 & ~15u);
					rs.kf_bit[1] += (tier_offset1 & 15u) * 8;
					rs.bit_base[1] = rs.kf_bit[1];
				}
			}
		}

		// seek_request of p.requests[request_index]. PAIRED: requests 2r and 2r + 1 are the two halves of pair r (additive or blend), sharing
		// the per request policies of pair r.
		template<bool DB = false, class RS = ReqState, bool PAIRED = false>
		__device__ __forceinline__ void seek_transform(const DecodeParams& p, uint32_t request_index, RS& rs)
		{
			seek_request<DB>(p, p.requests[request_index], PAIRED ? request_index >> 1 : request_index, rs);
		}

		// ---------------------------------------------------------------------------------------------------
		// bit stream reads. Streams are stored as byte-swapped 32-bit words (clipset.cpp append_stream): word i holds the
		// stream bits [32 i, 32 i + 32) MSB first, so the 32 bits that start at any bit are one funnel shift of two words.
		// ---------------------------------------------------------------------------------------------------
		template<bool STAGED, class RS>
		__device__ __forceinline__ uint32_t read_bits32(const RS& rs, const uint32_t* s_stage, int k, uint32_t bit_offset)
		{
			// unpack_vector3_96_unsafe, math/vector4_packing.h:482-503
			const uint32_t bit = rs.bit_base[k] + bit_offset;
			uint32_t hi, lo;
			if (STAGED)
			{
				const uint32_t* w = s_stage + rs.word_base[k] + (bit >> 5);
				hi = w[0];
				lo = w[1];
			}
			else
			{
				const uint32_t* w = reinterpret_cast<const uint32_t*>(stream_base(rs, k)) + (bit >> 5);
				hi = __ldg(w);
				lo = __ldg(w + 1);
			}
			return __funnelshift_l(lo, hi, bit & 31);
		}

		// quat_from_positive_w4, math/quatf.h:135-147
		__device__ __forceinline__ float quat_w(float x, float y, float z)
		{
			float r = fnegmulsub(x, x, 1.0f);
			r = fnegmulsub(y, y, r);
			r = fnegmulsub(z, z, r);
			return __fsqrt_rn(fabsf(r));
		}

		// quat_normalize4, math/quatf.h:200-211
		__device__ __forceinline__ void quat_normalize(float q[4])
		{
			float dot = fmul(q[0], q[0]);
			dot = fmuladd(q[1], q[1], dot);
			dot = fmuladd(q[2], q[2], dot);
			dot = fmuladd(q[3], q[3], dot);
			const float len = __fsqrt_rn(dot);
			const float inv_len = __frcp_rn(len);		// vector_div(1.0, len): a correctly rounded reciprocal
			q[0] = fmul(q[0], inv_len);
			q[1] = fmul(q[1], inv_len);
			q[2] = fmul(q[2], inv_len);
			q[3] = fmul(q[3], inv_len);
		}

		// quat_lerp_no_normalization4, math/quatf.h:170-196
		__device__ __forceinline__ void quat_lerp(const float s[4], const float e[4], float alpha, float out[4])
		{
			float dot = fmul(s[0], e[0]);
			dot = fmuladd(s[1], e[1], dot);
			dot = fmuladd(s[2], e[2], dot);
			dot = fmuladd(s[3], e[3], dot);
			const uint32_t bias = __float_as_uint(dot) & 0x80000000u;
#pragma unroll
			for (int i = 0; i < 4; ++i)
			{
				const float e_biased = __uint_as_float(__float_as_uint(e[i]) ^ bias);
				out[i] = fmuladd(e_biased, alpha, fnegmulsub(s[i], alpha, s[i]));
			}
		}

		// rtm::vector_lerp, external/rtm/includes/rtm/vector4f.h:2417-2421
		__device__ __forceinline__ float lerp(float start, float end, float alpha)
		{
			return fmuladd(end, alpha, fnegmulsub(start, alpha, start));
		}

		// rtm::quat_normalize (external/rtm/includes/rtm/quatf.h:917-953). On x86 this is rsqrtss + two Newton-Raphson steps,
		// whose result depends on the CPU's estimate table; we use the correctly rounded rsqrt, which every such estimate
		// converges to within 2 ulp (hence the 1e-5 gate on decompress_track rotations, SURVEY 8c).
		__device__ __forceinline__ void rtm_quat_normalize(float q[4])
		{
			const float x2 = fmul(q[0], q[0]), y2 = fmul(q[1], q[1]), z2 = fmul(q[2], q[2]), w2 = fmul(q[3], q[3]);
			const float dot = fadd(fadd(x2, z2), fadd(y2, w2));
			const float inv_len = __frsqrt_rn(dot);
#pragma unroll
			for (int i = 0; i < 4; ++i)
				q[i] = fmul(q[i], inv_len);
		}

		// rtm::quat_lerp / acl::quat_lerp_no_normalization, SSE4 flavour (dpps sums (x+y)+(z+w)),
		// external/rtm/includes/rtm/quatf.h:1006-1075, math/quatf.h:40-82
		__device__ __forceinline__ void rtm_quat_lerp(const float s[4], const float e[4], float alpha, bool normalize, float out[4])
		{
			const float dot = fadd(fadd(fmul(s[0], e[0]), fmul(s[1], e[1])), fadd(fmul(s[2], e[2]), fmul(s[3], e[3])));
			const uint32_t bias = __float_as_uint(dot) & 0x80000000u;
#pragma unroll
			for (int i = 0; i < 4; ++i)
				out[i] = fadd(fsub(s[i], fmul(alpha, s[i])), fmul(alpha, __uint_as_float(__float_as_uint(e[i]) ^ bias)));
			if (normalize)
				rtm_quat_normalize(out);
		}

		// ---------------------------------------------------------------------------------------------------
		// sub-track decoders
		// ---------------------------------------------------------------------------------------------------
		__device__ __forceinline__ Entry entry_from(const uint4& v)
		{
			Entry e;
			e.offset_code = v.x; e.inv_max = __uint_as_float(v.y);
			e.range_lo = v.z; e.range_hi = v.w;
			return e;
		}

		__device__ __forceinline__ Entry load_entry(const ReqState& rs, int k, uint32_t slot)
		{
			return entry_from(__ldg(reinterpret_cast<const uint4*>(rs.image + rs.entries_off[k]) + slot));
		}

		// Segment range byte `i` (0..3) of `word` expanded as unpack_segment_range_data does (animated_track_cache.transform.h:157-298):
		// u8 -> float, times 1 / 255 in float. The conversion is exact either way; here it is one byte permute into the mantissa of 2^23
		// and one subtraction, both full rate.
		__device__ __forceinline__ float range_byte(uint32_t word, uint32_t i)
		{
			const float biased = __uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440u | i));		// 2^23 + byte
			return fmul(fsub(biased, 8388608.0f), 1.0f / 255.0f);
		}
		// the segment range of a quantised Entry (codes 1..23): lo = Entry::range_lo, hi = Entry::range_hi
		__device__ __forceinline__ float range_min_x(uint32_t lo) { return range_byte(lo, 0); }
		__device__ __forceinline__ float range_min_y(uint32_t lo) { return range_byte(lo, 1); }
		__device__ __forceinline__ float range_min_z(uint32_t lo) { return range_byte(lo, 2); }
		__device__ __forceinline__ float range_extent_x(uint32_t lo) { return range_byte(lo, 3); }
		__device__ __forceinline__ float range_extent_y(uint32_t hi) { return range_byte(hi, 0); }
		__device__ __forceinline__ float range_extent_z(uint32_t hi) { return range_byte(hi, 1); }

		// Raw integers of one animated sample: x, y, z (quantised integers or raw float bits), shared by the decode and by the
		// parity hook (unpack_animated_quat / unpack_animated_vector3 integer stage).
		template<bool STAGED, class RS>
		__device__ __forceinline__ void unpack_sample_ints(const RS& rs, const uint32_t* s_stage, int k, const Entry& e, bool four_components,
			uint32_t& xi, uint32_t& yi, uint32_t& zi, uint32_t& wi)
		{
			const uint32_t code = e.offset_code & 0xFFu;
			const uint32_t bit_offset = e.offset_code >> 8;
			wi = 0;
			if (code == 0)
			{
				// constant inside the segment: the 3 x 16 bit sample was gathered from the segment range bytes at upload
				// (animated_track_cache.transform.h:552-587; unpack_vector3_u48_unsafe, math/vector4_packing.h:628-653)
				xi = e.range_lo & 0xFFFFu;
				yi = e.range_lo >> 16;
				zi = e.range_hi & 0xFFFFu;
			}
			else if (code & k_entry_raw)
			{
				xi = read_bits32<STAGED>(rs, s_stage, k, bit_offset);
				yi = read_bits32<STAGED>(rs, s_stage, k, bit_offset + 32);
				zi = read_bits32<STAGED>(rs, s_stage, k, bit_offset + 64);
				if (four_components)
					wi = read_bits32<STAGED>(rs, s_stage, k, bit_offset + 96);
			}
			else
			{
				// unpack_vector3_uXX_unsafe, math/vector4_packing.h:947-971
				const uint32_t shift = 32 - code;
				xi = read_bits32<STAGED>(rs, s_stage, k, bit_offset) >> shift;
				yi = read_bits32<STAGED>(rs, s_stage, k, bit_offset + code) >> shift;
				zi = read_bits32<STAGED>(rs, s_stage, k, bit_offset + code * 2) >> shift;
			}
		}

		// One animated rotation sample after range expansion and W reconstruction.
		// SINGLE == false: decompress_tracks flavour (unpack_animated_quat + remap_segment_range_data4 + remap_clip_range_data4,
		//                  animated_track_cache.transform.h:515-687,302-350,391-466): ignored ranges still multiply by 1 and add 0.
		// SINGLE == true : decompress_track flavour (unpack_single_animated_quat, :689-869): ignored ranges are skipped.
		template<bool SINGLE, bool STAGED, class RS>
		__device__ __forceinline__ void decode_animated_rotation(const RS& rs, const uint32_t* s_stage, int k, const Entry& e,
			const float4& clip_extent, const float4& clip_min, float out[4])
		{
			const bool rot_full = (rs.clip_flags & k_clip_rot_full) != 0;
			uint32_t xi, yi, zi, wi;
			unpack_sample_ints<STAGED>(rs, s_stage, k, e, rot_full, xi, yi, zi, wi);
			const uint32_t code = e.offset_code & 0xFFu;

			if (!(rs.clip_flags & k_clip_rot_variable))
			{
				out[0] = __uint_as_float(xi);
				out[1] = __uint_as_float(yi);
				out[2] = __uint_as_float(zi);
				out[3] = rot_full ? __uint_as_float(wi) : quat_w(out[0], out[1], out[2]);
				return;
			}

			float x, y, z;
			const bool is_raw = (code & k_entry_raw) != 0;
			const bool ignore_segment = code == 0 || is_raw;
			const bool ignore_clip = is_raw;
			if (is_raw)
			{
				x = __uint_as_float(xi); y = __uint_as_float(yi); z = __uint_as_float(zi);
			}
			else
			{
				// code 0: 1 / 65535, else 1 / (2^code - 1) -- both stored in the entry
				x = fmul(u2f(xi), e.inv_max); y = fmul(u2f(yi), e.inv_max); z = fmul(u2f(zi), e.inv_max);
			}

			if ((rs.clip_flags & k_clip_has_segments) && (!SINGLE || !ignore_segment))
			{
				// unpack_segment_range_data, :157-298: u8 * (1 / 255); a constant sample (its range bytes hold the sample integers) and a
				// raw one take min = 0, extent = 1
				x = fmuladd(x, ignore_segment ? 1.0f : range_extent_x(e.range_lo), ignore_segment ? 0.0f : range_min_x(e.range_lo));
				y = fmuladd(y, ignore_segment ? 1.0f : range_extent_y(e.range_hi), ignore_segment ? 0.0f : range_min_y(e.range_lo));
				z = fmuladd(z, ignore_segment ? 1.0f : range_extent_z(e.range_hi), ignore_segment ? 0.0f : range_min_z(e.range_lo));
			}

			if (!SINGLE || !ignore_clip)
			{
				// remap_clip_range_data4, :391-466
				const float ext_x = ignore_clip ? 1.0f : clip_extent.x, ext_y = ignore_clip ? 1.0f : clip_extent.y, ext_z = ignore_clip ? 1.0f : clip_extent.z;
				const float min_x = ignore_clip ? 0.0f : clip_min.x, min_y = ignore_clip ? 0.0f : clip_min.y, min_z = ignore_clip ? 0.0f : clip_min.z;
				x = fmuladd(x, ext_x, min_x);
				y = fmuladd(y, ext_y, min_y);
				z = fmuladd(z, ext_z, min_z);
			}

			out[0] = x; out[1] = y; out[2] = z;
			out[3] = quat_w(x, y, z);
		}

		// unpack_animated_vector3 / unpack_single_animated_vector3, animated_track_cache.transform.h:871-990,992-1102
		template<bool STAGED, class RS>
		__device__ __forceinline__ void decode_animated_vector3(const RS& rs, const uint32_t* s_stage, int k, const Entry& e, bool variable,
			const float4& clip_extent, const float4& clip_min, float out[3])
		{
			uint32_t xi, yi, zi, wi;
			unpack_sample_ints<STAGED>(rs, s_stage, k, e, false, xi, yi, zi, wi);
			const uint32_t code = e.offset_code & 0xFFu;

			if (!variable || (code & k_entry_raw))
			{
				out[0] = __uint_as_float(xi); out[1] = __uint_as_float(yi); out[2] = __uint_as_float(zi);
				return;
			}

			float x = fmul(u2f(xi), e.inv_max), y = fmul(u2f(yi), e.inv_max), z = fmul(u2f(zi), e.inv_max);
			if (code != 0 && (rs.clip_flags & k_clip_has_segments))
			{
				// unpack_vector3_u24_unsafe min then extent, math/vector4_packing.h:781-818
				x = fmuladd(x, range_extent_x(e.range_lo), range_min_x(e.range_lo));
				y = fmuladd(y, range_extent_y(e.range_hi), range_min_y(e.range_lo));
				z = fmuladd(z, range_extent_z(e.range_hi), range_min_z(e.range_lo));
			}
			// clip range (:949-958)
			out[0] = fmuladd(x, clip_extent.x, clip_min.x);
			out[1] = fmuladd(y, clip_extent.y, clip_min.y);
			out[2] = fmuladd(z, clip_extent.z, clip_min.z);
		}

		// should_interpolate_samples, decompression_context.transform.h:191-200
		__device__ __forceinline__ bool should_interpolate(const DecodeParams& p, uint32_t clip_flags, float alpha)
		{
			if (p.multiple_rotation_formats)
				return true;
			return (clip_flags & k_clip_rot_full) ? (alpha > 0.0f && alpha < 1.0f) : true;
		}

		__device__ __forceinline__ uint32_t track_rounding_policy(const DecodeParams& p, uint32_t track)
		{
			// track_writer::get_rounding_policy(seek_policy, track_index), core/track_writer.h:90
			if (p.rounding_policy != ACLB200_ROUND_PER_TRACK || p.per_track_policies == nullptr)
				return p.rounding_policy;
			return p.per_track_policies[track];
		}

		// Default sub-tracks: unpack_default_*_sub_tracks, decompression.transform.h:574-675,881-983,1201-1310. writer_defaults: the
		// acl::track_writer defaults whatever the options say (core/track_writer.h:160-176): constant identity rotation, constant zero
		// translation, legacy scale -- what a default sub-track of an additive clip means.
		__device__ __forceinline__ bool default_value(const DecodeParams& p, uint32_t kind, uint32_t track, uint32_t clip_flags, float out[4],
			bool writer_defaults = false)
		{
			if (writer_defaults)
			{
				const float s = kind == 2 && (clip_flags & k_clip_default_scale_one) ? 1.0f : 0.0f;
				out[0] = s; out[1] = s; out[2] = s; out[3] = kind == 0 ? 1.0f : s;
				return true;
			}
			const uint32_t mode = p.default_mode[kind];
			if (mode == ACLB200_DEFAULT_SKIPPED)
				return false;
			if (mode == ACLB200_DEFAULT_VARIABLE && p.variable_defaults != nullptr)
			{
				const float* v = p.variable_defaults + size_t(track) * 12 + kind * 4;
				out[0] = v[0]; out[1] = v[1]; out[2] = v[2]; out[3] = v[3];
			}
			else if (mode == ACLB200_DEFAULT_LEGACY && kind == 2)
			{
				const float s = (clip_flags & k_clip_default_scale_one) ? 1.0f : 0.0f;	// float(header.get_default_scale()), :1548
				out[0] = s; out[1] = s; out[2] = s; out[3] = s;
			}
			else
			{
				out[0] = p.constant_defaults[kind * 4 + 0]; out[1] = p.constant_defaults[kind * 4 + 1];
				out[2] = p.constant_defaults[kind * 4 + 2]; out[3] = p.constant_defaults[kind * 4 + 3];
			}
			return true;
		}

		// ---- the device track_writer: write_rotation / write_translation / write_scale ----
		__device__ __forceinline__ void write_rotation(uint32_t layout, uint8_t* bone, const float q[4])
		{
			if (layout == ACLB200_LAYOUT_QVV48)
				*reinterpret_cast<float4*>(bone) = make_float4(q[0], q[1], q[2], q[3]);
			else
			{
				float2* dst = reinterpret_cast<float2*>(bone);		// 40 byte bones are 8 byte aligned
				dst[0] = make_float2(q[0], q[1]);
				dst[1] = make_float2(q[2], q[3]);
			}
		}

		__device__ __forceinline__ void write_vector(uint32_t layout, uint8_t* bone, uint32_t kind, const float v[3])
		{
			if (layout == ACLB200_LAYOUT_QVV48)
				*reinterpret_cast<float4*>(bone + 16 * kind) = make_float4(v[0], v[1], v[2], 0.0f);
			else if (kind == 1)
			{
				*reinterpret_cast<float2*>(bone + 16) = make_float2(v[0], v[1]);
				*reinterpret_cast<float*>(bone + 24) = v[2];
			}
			else
			{
				*reinterpret_cast<float*>(bone + 28) = v[0];
				*reinterpret_cast<float2*>(bone + 32) = make_float2(v[1], v[2]);
			}
		}

		// Interpolation of two decoded rotation samples: unpack_rotation_group, animated_track_cache.transform.h:1463-1474,1477-1661
		// (SINGLE: unpack_rotation_within_group, :1709-1765)
		template<int NORM, bool PER_TRACK, bool SINGLE>
		__device__ __forceinline__ void interpolate_rotation(const DecodeParams& p, uint32_t clip_flags, float s0[4], float s1[4], float alpha, uint32_t policy, float rotation[4])
		{
			const bool interpolate = should_interpolate(p, clip_flags, alpha);
			if (SINGLE)
			{
				if (interpolate)
					rtm_quat_lerp(s0, s1, alpha, NORM >= ACLB200_NORMALIZE_LERP_ONLY, rotation);
				else
				{
#pragma unroll
					for (int i = 0; i < 4; ++i)
						rotation[i] = alpha <= 0.0f ? s0[i] : s1[i];
					if (NORM == ACLB200_NORMALIZE_ALWAYS && !(clip_flags & k_clip_rot_full))
						rtm_quat_normalize(rotation);
				}
				return;
			}

			if (NORM == ACLB200_NORMALIZE_ALWAYS && !(clip_flags & k_clip_rot_full) && (PER_TRACK || !interpolate))
			{
				quat_normalize(s0);
				quat_normalize(s1);
			}

			if (PER_TRACK && policy == ACLB200_ROUND_FLOOR)
			{
#pragma unroll
				for (int i = 0; i < 4; ++i) rotation[i] = s0[i];
			}
			else if (PER_TRACK && policy == ACLB200_ROUND_CEIL)
			{
#pragma unroll
				for (int i = 0; i < 4; ++i) rotation[i] = s1[i];
			}
			else if (PER_TRACK && policy == ACLB200_ROUND_NEAREST)
			{
#pragma unroll
				for (int i = 0; i < 4; ++i) rotation[i] = alpha < 0.5f ? s0[i] : s1[i];
			}
			else if (PER_TRACK || interpolate)
			{
				quat_lerp(s0, s1, alpha, rotation);
				if (NORM >= ACLB200_NORMALIZE_LERP_ONLY)
					quat_normalize(rotation);
			}
			else
			{
#pragma unroll
				for (int i = 0; i < 4; ++i) rotation[i] = alpha <= 0.0f ? s0[i] : s1[i];
			}
		}

		// One animated rotation sub-track of one request (phase 3)
		template<int NORM, bool PER_TRACK, bool SINGLE, bool STAGED, class RS>
		__device__ __forceinline__ uint32_t animated_rotation(const DecodeParams& p, const RS& rs, const uint32_t* s_stage, uint32_t rank, float alpha_in, float rotation[4])
		{
			const float4* anim = reinterpret_cast<const float4*>(rs.image + rs.anim_off) + rank;
			const float4 clip_extent = __ldg(anim);		// .w carries the bone index
			const float4 clip_min = __ldg(anim + (rs.num_animated[0] + rs.num_animated[1] + rs.num_animated[2]));
			const uint32_t bone = __float_as_uint(clip_extent.w);
			const Entry e0 = load_entry(rs, 0, rank);
			const Entry e1 = rs.single_segment ? e0 : load_entry(rs, 1, rank);

			float s0[4], s1[4];
			decode_animated_rotation<SINGLE, STAGED>(rs, s_stage, 0, e0, clip_extent, clip_min, s0);
			decode_animated_rotation<SINGLE, STAGED>(rs, s_stage, 1, e1, clip_extent, clip_min, s1);

			const uint32_t policy = PER_TRACK ? track_rounding_policy(p, bone) : ACLB200_ROUND_NONE;
			const float alpha = (SINGLE && PER_TRACK) ? apply_rounding_policy(alpha_in, policy) : alpha_in;	// :1975-1983
			interpolate_rotation<NORM, PER_TRACK, SINGLE>(p, rs.clip_flags, s0, s1, alpha, policy, rotation);
			return bone;
		}

		// One animated translation (kind 1) or scale (kind 2) sub-track of one request (phase 4):
		// unpack_translation_group / consume_translation, animated_track_cache.transform.h:1774-1836,1889-1894
		template<bool PER_TRACK, bool SINGLE, bool STAGED, class RS>
		__device__ __forceinline__ uint32_t animated_vector(const DecodeParams& p, const RS& rs, const uint32_t* s_stage, uint32_t kind, uint32_t rank, float alpha_in, float value[3])
		{
			const uint32_t slot = rs.num_animated[0] + (kind == 2 ? rs.num_animated[1] : 0u) + rank;
			const float4* anim = reinterpret_cast<const float4*>(rs.image + rs.anim_off) + slot;
			const float4 clip_extent = __ldg(anim);
			const float4 clip_min = __ldg(anim + (rs.num_animated[0] + rs.num_animated[1] + rs.num_animated[2]));
			const uint32_t bone = __float_as_uint(clip_extent.w);
			const Entry e0 = load_entry(rs, 0, slot);
			const Entry e1 = rs.single_segment ? e0 : load_entry(rs, 1, slot);
			const bool variable = (rs.clip_flags & (kind == 1 ? k_clip_trans_variable : k_clip_scale_variable)) != 0;

			float s0[3], s1[3];
			decode_animated_vector3<STAGED>(rs, s_stage, 0, e0, variable, clip_extent, clip_min, s0);
			decode_animated_vector3<STAGED>(rs, s_stage, 1, e1, variable, clip_extent, clip_min, s1);

			const uint32_t policy = PER_TRACK ? track_rounding_policy(p, bone) : ACLB200_ROUND_NONE;
			const float alpha = (SINGLE && PER_TRACK) ? apply_rounding_policy(alpha_in, policy) : alpha_in;
#pragma unroll
			for (int i = 0; i < 3; ++i)
			{
				if (!SINGLE && PER_TRACK && policy == ACLB200_ROUND_FLOOR)
					value[i] = s0[i];
				else if (!SINGLE && PER_TRACK && policy == ACLB200_ROUND_CEIL)
					value[i] = s1[i];
				else if (!SINGLE && PER_TRACK && policy == ACLB200_ROUND_NEAREST)
					value[i] = alpha < 0.5f ? s0[i] : s1[i];
				else
					value[i] = lerp(s0[i], s1[i], alpha);
			}
			return bone;
		}

		// Constant and default sub-tracks of one bone (phase 2): unpack_default_* / unpack_constant_*_sub_tracks,
		// decompression.transform.h:574-748,881-1072,1201-1430; constant rotations had their W reconstructed (and normalised) at upload
		// (writer_defaults: see default_value)
		template<int NORM, bool SINGLE>
		__device__ __forceinline__ void constant_sub_tracks(const DecodeParams& p, const ReqState& rs, uint32_t bone, uint64_t desc, uint8_t* out_bone,
			bool writer_defaults = false)
		{
			// rotation
			{
				const uint32_t type = uint32_t(desc) & 3;
				const uint32_t rank = (uint32_t(desc) >> 2) & k_bone_index_mask;
				float q[4];
				if (skip_sub_track(p, 0, bone))
				{
				}
				else if (type == 0)
				{
					if (default_value(p, 0, bone, rs.clip_flags, q, writer_defaults))
						write_rotation(p.layout, out_bone, q);
				}
				else if (type == 1)
				{
					const float4* table = reinterpret_cast<const float4*>(rs.image + rs.const_rot_off) + size_t(rank) * 2;
					if (SINGLE && NORM == ACLB200_NORMALIZE_ALWAYS && !(rs.clip_flags & k_clip_rot_full))
					{
						// unpack_rotation_within_group normalises with rtm::quat_normalize, constant_track_cache.transform.h:255-258
						const float4 v = __ldg(table);
						q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
						rtm_quat_normalize(q);
					}
					else
					{
						const float4 v = __ldg(table + (NORM == ACLB200_NORMALIZE_ALWAYS ? 1 : 0));
						q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
					}
					write_rotation(p.layout, out_bone, q);
				}
			}
			// translation, scale
#pragma unroll
			for (uint32_t kind = 1; kind <= 2; ++kind)
			{
				const uint32_t bits = uint32_t(desc >> (k_bone_kind_shift * kind));
				// clips without scale: every bone takes the default (decompression.transform.h:1653-1680,1806-1822)
				const uint32_t type = (kind == 2 && !(rs.clip_flags & k_clip_has_scale)) ? 0u : (bits & 3);
				const uint32_t rank = (bits >> 2) & k_bone_index_mask;
				float v[4];
				if (skip_sub_track(p, kind, bone))
					continue;
				if (type == 0)
				{
					if (default_value(p, kind, bone, rs.clip_flags, v, writer_defaults))
						write_vector(p.layout, out_bone, kind, v);
				}
				else if (type == 1)
				{
					const float4 c = __ldg(reinterpret_cast<const float4*>(rs.image + rs.const_vec_off) + (kind == 2 ? rs.num_constant_trans : 0u) + rank);
					v[0] = c.x; v[1] = c.y; v[2] = c.z;
					write_vector(p.layout, out_bone, kind, v);
				}
			}
		}

		// One bone's row of a request for the launches that decode a few bones of each request (the bone query's closure, root motion's
		// root): its three sub-tracks one after the other, key frames read from global memory, with the plain kernel's decoders
		// (SINGLE = false). Those entry points refuse skip masks, so the animated sub-tracks are not checked against them: the checks made
		// both routes 0.2 to 1 % slower (H100). decompress_track's kernel honours skip masks and keeps its own copy of this sequence.
		template<int NORM, bool PER_TRACK, class RS>
		__device__ __forceinline__ void decode_bone_row(const DecodeParams& p, const RS& rs, uint32_t bone, uint8_t* out_bone)
		{
			const uint64_t desc = __ldg(reinterpret_cast<const unsigned long long*>(rs.image + rs.bone_table_off) + bone);
			constant_sub_tracks<NORM, false>(p, rs, bone, desc, out_bone);
			if ((uint32_t(desc) & 3) == 2)
			{
				float rotation[4];
				animated_rotation<NORM, PER_TRACK, false, false>(p, rs, nullptr, (uint32_t(desc) >> 2) & k_bone_index_mask, rs.alpha, rotation);
				write_rotation(p.layout, out_bone, rotation);
			}
#pragma unroll
			for (uint32_t kind = 1; kind <= 2; ++kind)
			{
				const uint32_t bits = uint32_t(desc >> (k_bone_kind_shift * kind));
				if ((bits & 3) == 2 && (kind == 1 || (rs.clip_flags & k_clip_has_scale)))
				{
					float value[3];
					animated_vector<PER_TRACK, false, false>(p, rs, nullptr, kind, (bits >> 2) & k_bone_index_mask, rs.alpha, value);
					write_vector(p.layout, out_bone, kind, value);
				}
			}
		}

		__device__ __forceinline__ uint32_t fast_div(uint32_t value, uint32_t magic)
		{
			return magic != 0 ? __umulhi(value, magic) : value;
		}

	}
}
