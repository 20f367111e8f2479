// acl_b200/csrc/clipset.cpp -- host side of aclb200_upload_clips: validate the caller's compressed_tracks blobs and
// transcode each one into the GPU-native clip image described in layout.h.
//
// This is the batched counterpart of decompression_context::initialize()
// (includes/acl/decompression/impl/decompress.impl.h:66-83 -> initialize_v0,
// includes/acl/decompression/impl/decompression.transform.h:84-132 / decompression.scalar.h:99-123). The reference
// caches a handful of header fields per context and re-derives everything else on every seek with serial cursors; a
// GPU thread cannot run those cursors, so the offsets, ranks and per sub-track bit positions are tabulated here once.
// Float values computed here (W of constant rotations, 1/(2^n - 1)) use the same IEEE-754 single precision operations
// in the same order as the reference's decoder, so nothing about the results changes.
#include "context.h"

#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <limits>
#include <new>
#include <thread>
#if defined(__linux__)
#include <sched.h>
#endif

namespace aclb200
{
	namespace
	{
		inline uint32_t rd_u32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
		inline uint16_t rd_u16(const uint8_t* p) { uint16_t v; std::memcpy(&v, p, 2); return v; }
		inline float rd_f32(const uint8_t* p) { float v; std::memcpy(&v, p, 4); return v; }
		inline uint32_t align_up(uint32_t v, uint32_t a) { return (v + a - 1) & ~(a - 1); }
		inline uint64_t align_up64(uint64_t v, uint64_t a) { return (v + a - 1) & ~(a - 1); }

		// core/hash.h:44-84 (FNV-1a 32), the hash compressed_tracks::is_valid(true) verifies
		uint32_t hash32(const uint8_t* data, size_t size)
		{
			uint32_t acc = 2166136261u;
			for (size_t i = 0; i < size; ++i)
				acc = (acc ^ data[i]) * 16777619u;
			return acc;
		}

		// core/impl/variable_bit_rates.h:39-43
		const uint8_t k_bit_rate_num_bits_v0[] = { 0, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 32 };
		const uint8_t k_bit_rate_num_bits[] = { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 32 };

		// calculate_finite_duration, core/impl/time_utils.impl.h:105-114
		float finite_duration(uint32_t num_samples, float sample_rate)
		{
			if (num_samples <= 1)
				return 0.0F;
			return float(num_samples - 1) / sample_rate;
		}

		// PackedTableEntry::max_value, math/vector4_packing.h:927-929: a float division evaluated in float
		float inv_max_value(uint32_t num_bits)
		{
			return 1.0F / float((1u << num_bits) - 1u);
		}

		struct image_too_large {};

		// Growable clip image with 16 byte aligned sections
		struct image_builder
		{
			std::vector<uint8_t>& bytes;
			size_t base;
			explicit image_builder(std::vector<uint8_t>& bytes_) : bytes(bytes_), base(bytes_.size()) {}
			// image offsets are 32 bit: a clip whose image would pass 4 GiB is refused (image_too_large, caught by build_clipset), never wrapped
			uint32_t reserve(size_t size)
			{
				const size_t offset = align_up64(bytes.size() - base, k_section_alignment);
				if (offset + size > 0xFFFFFFF0ull)
					throw image_too_large();
				bytes.resize(base + offset + size, 0);
				return uint32_t(offset);
			}
			uint8_t* at(uint32_t offset) { return bytes.data() + base + offset; }
		};

		// Copies `num_bytes` of a big-endian bit stream as byte-swapped 32-bit words (so word i holds stream bits [32 i, 32 i + 32)
		// with bit 0 of the stream in the MSB) and leaves k_stream_tail zero bytes behind it.
		uint32_t append_stream(image_builder& image, const uint8_t* src, size_t num_bytes)
		{
			const size_t padded = align_up64(num_bytes, 4);
			const uint32_t offset = image.reserve(padded + k_stream_tail);
			uint8_t* dst = image.at(offset);
			for (size_t i = 0; i < num_bytes; ++i)
				dst[(i & ~size_t(3)) + (3 - (i & 3))] = src[i];
			return offset;
		}

		struct parse_result
		{
			ClipDesc desc;
			uint32_t looping_policy;
			uint32_t track_type;
			uint32_t max_key_frame_bytes;
			uint32_t db_clip_header_offset;		// tracks_database_header::clip_header_offset, 0xFFFFFFFF without a database
			std::vector<uint32_t> db_pose_bits;	// animated_pose_bit_size per segment of a clip bound to a database
		};

		// Validates one blob and appends its clip image to `data`. Returns an empty string on success, else why the clip is
		// rejected; `unsupported` tells apart valid ACL data we refuse (unknown track types, images past 4 GiB) from invalid buffers.
		std::string transcode_clip(const uint8_t* blob, uint32_t size, bool check_hash, std::vector<uint8_t>& data, parse_result& out, bool& unsupported)
		{
			unsupported = false;

			// compressed_tracks::is_valid, core/impl/compressed_tracks.impl.h:278-301
			if (blob == nullptr || size < k_type_header_offset + 20)
				return "buffer too small";
			const uint32_t stored_size = rd_u32(blob + 0);
			if (stored_size > size || stored_size < k_type_header_offset + 20)
				return "stored size does not fit the buffer";
			if (rd_u32(blob + 8) != k_tag)
				return "invalid tag";
			const uint32_t version = rd_u16(blob + 12);
			if (blob[14] != 0)
				return "invalid algorithm type";
			if (version < k_version_first || version > k_version_latest)
				return "invalid algorithm version";
			if (check_hash && hash32(blob + 8, stored_size - 8) != rd_u32(blob + 4))
				return "invalid hash";

			const uint32_t track_type = blob[15];
			const uint32_t num_tracks = rd_u32(blob + 16);
			const uint32_t num_samples = rd_u32(blob + 20);
			const float sample_rate = rd_f32(blob + 24);
			const uint32_t misc = rd_u32(blob + 28);
			const bool is_wrap = version > k_version_first && ((misc >> 30) & 1) != 0;	// compressed_tracks.impl.h:127-134

			if (track_type != k_track_qvvf && track_type > 4)
				return "unsupported track type";
			if (num_tracks > k_max_tracks)
			{
				unsupported = true;
				return "too many tracks for the bone index table";
			}

			ClipDesc& d = out.desc;
			std::memset(&d, 0, sizeof(d));
			d.num_tracks = num_tracks;
			d.num_samples = num_samples;
			d.sample_rate = sample_rate;
			d.duration_clamp = finite_duration(num_samples, sample_rate);
			d.duration_wrap = finite_duration(num_samples != 0 ? num_samples + 1 : 0, sample_rate);
			d.hash = rd_u32(blob + 4);
			d.size = stored_size;
			out.looping_policy = is_wrap ? ACLB200_LOOP_WRAP : ACLB200_LOOP_CLAMP;
			out.track_type = track_type;
			out.max_key_frame_bytes = 0;
			out.db_clip_header_offset = 0xFFFFFFFFu;
			out.db_pose_bits.clear();
			if (is_wrap)
				d.flags |= k_clip_wrap;

			image_builder image(data);
			const uint8_t* th = blob + k_type_header_offset;
			auto in_bounds = [&](uint64_t offset_from_blob, uint64_t bytes) { return offset_from_blob + bytes <= stored_size; };

			if (track_type != k_track_qvvf)
			{
				// scalar_tracks_header, core/impl/compressed_headers.h:140-165; stream writers compress.scalar.impl.h:93-175
				const uint32_t num_bits_per_frame = rd_u32(th + 0);
				const uint32_t metadata_offset = k_type_header_offset + rd_u32(th + 4);
				const uint32_t constant_offset = k_type_header_offset + rd_u32(th + 8);
				const uint32_t range_offset = k_type_header_offset + rd_u32(th + 12);
				const uint32_t animated_offset = k_type_header_offset + rd_u32(th + 16);
				if (num_tracks != 0 && !in_bounds(metadata_offset, num_tracks))
					return "track metadata out of bounds";

				const uint32_t num_components = track_type <= 3 ? track_type + 1 : 4;
				const uint8_t* table = version == k_version_first ? k_bit_rate_num_bits_v0 : k_bit_rate_num_bits;
				const uint32_t table_size = version == k_version_first ? sizeof(k_bit_rate_num_bits_v0) : sizeof(k_bit_rate_num_bits);

				d.bone_table_offset = image.reserve(size_t(num_tracks) * sizeof(ScalarTrackDesc));
				uint32_t bit_offset = 0, constant_index = 0, range_index = 0;
				for (uint32_t track = 0; track < num_tracks; ++track)
				{
					const uint32_t bit_rate = blob[metadata_offset + track];
					if (bit_rate >= table_size)
						return "invalid scalar bit rate";
					const uint32_t num_bits = table[bit_rate];
					ScalarTrackDesc desc = {};
					desc.bit_offset = bit_offset;
					desc.inv_max = 1.0F;
					if (num_bits == 0)
					{
						desc.value_index_and_bits = (constant_index << 8) | 0u;
						constant_index += num_components;
					}
					else if (num_bits == 32)
						desc.value_index_and_bits = 32u;
					else
					{
						desc.value_index_and_bits = (range_index << 8) | num_bits;
						desc.inv_max = inv_max_value(num_bits);
						range_index += num_components * 2;
					}
					std::memcpy(image.at(d.bone_table_offset) + size_t(track) * sizeof(ScalarTrackDesc), &desc, sizeof(desc));
					bit_offset += num_bits * num_components;
				}
				if (bit_offset != num_bits_per_frame)
					return "scalar bit rates do not add up to num_bits_per_frame";
				if (!in_bounds(constant_offset, uint64_t(constant_index) * 4) || !in_bounds(range_offset, uint64_t(range_index) * 4))
					return "scalar constant / range values out of bounds";
				const uint64_t stream_bytes = (uint64_t(num_bits_per_frame) * num_samples + 7) / 8;
				if (num_samples != 0 && !in_bounds(animated_offset, stream_bytes))
					return "scalar animated values out of bounds";

				d.const_rot_offset = image.reserve(size_t(constant_index) * 4 + 16);
				std::memcpy(image.at(d.const_rot_offset), blob + constant_offset, size_t(constant_index) * 4);
				d.const_vec_offset = image.reserve(size_t(range_index) * 4 + 16);
				std::memcpy(image.at(d.const_vec_offset), blob + range_offset, size_t(range_index) * 4);
				// the same values once more, indexed by track: min[components], extent[components]
				d.track_range_offset = image.reserve(size_t(num_tracks) * num_components * 8 + 16);
				for (uint32_t track = 0; track < num_tracks; ++track)
				{
					ScalarTrackDesc desc;
					std::memcpy(&desc, image.at(d.bone_table_offset) + size_t(track) * sizeof(ScalarTrackDesc), sizeof(desc));
					const uint32_t num_bits = desc.value_index_and_bits & 0xFFu, value_index = desc.value_index_and_bits >> 8;
					float* row = reinterpret_cast<float*>(image.at(d.track_range_offset)) + size_t(track) * num_components * 2;
					for (uint32_t c = 0; c < num_components; ++c)
					{
						if (num_bits == 0)
						{
							row[c] = rd_f32(blob + constant_offset + (value_index + c) * 4);
							row[num_components + c] = 0.0F;
						}
						else if (num_bits == 32)
						{
							row[c] = 0.0F;
							row[num_components + c] = 1.0F;
						}
						else
						{
							row[c] = rd_f32(blob + range_offset + (value_index + c) * 4);
							row[num_components + c] = rd_f32(blob + range_offset + (value_index + num_components + c) * 4);
						}
					}
				}
				d.seg_table_offset = append_stream(image, blob + animated_offset, size_t(stream_bytes));

				d.num_segments = 1;
				d.samples_per_segment = num_samples;
				d.num_animated_total = num_bits_per_frame;
				out.max_key_frame_bytes = (num_bits_per_frame + 7) / 8;
				d.image_size = image.reserve(0);
				return std::string();
			}

			// ---- transform clips: tracks_header::misc_packed accessors, compressed_headers.h:95-124 ----
			if (!in_bounds(k_type_header_offset, k_transform_header_size))
				return "transform header out of bounds";
			const bool has_scale = (misc & 1) != 0;
			const uint32_t scale_format = (misc >> 2) & 1;
			const uint32_t translation_format = (misc >> 3) & 1;
			const uint32_t rotation_format = (misc >> 4) & 15;
			const bool has_database = ((misc >> 8) & 1) != 0;
			// A clip bound to a streaming database (SURVEY 8 f2) is decoded from the key frames that stay resident in the clip until its
			// clip set is bound to the database and tiers are streamed in (database.cpp): what decompression_context<settings with
			// database support>::initialize(tracks) gives with no database bound, and with a database none of whose tiers is streamed in
			// (decompress.impl.h:67-83; seek_v0 treats it as a clip with stripped key frames, decompression.transform.h:262-265). Its
			// transform header names the database metadata (compressed_headers.h:245-246): the flag without that header is a corrupt clip.
			if (has_database)
			{
				const uint32_t database_header_offset = rd_u32(blob + k_type_header_offset + 32);
				if (database_header_offset == 0xFFFFFFFFu || !in_bounds(k_type_header_offset + database_header_offset, 8))
					return "database flag without a database header";
				out.db_clip_header_offset = rd_u32(blob + k_type_header_offset + database_header_offset);
			}
			const bool has_stripped = ((misc >> 10) & 1) != 0 || has_database;
			if (rotation_format != k_rot_full && rotation_format != k_rot_drop_w_full && rotation_format != k_rot_drop_w_variable)
				return "invalid rotation format";

			// transform_tracks_header, compressed_headers.h:227-262
			const uint32_t num_segments = rd_u32(th + 0);
			const uint32_t num_variable = rd_u32(th + 4);
			const uint32_t num_animated[3] = { rd_u32(th + 8), rd_u32(th + 12), has_scale ? rd_u32(th + 16) : 0u };
			const uint32_t num_constant[3] = { rd_u32(th + 20), rd_u32(th + 24), has_scale ? rd_u32(th + 28) : 0u };
			const uint32_t segment_headers_offset = k_type_header_offset + rd_u32(th + 36);
			const uint32_t sub_track_types_offset = k_type_header_offset + rd_u32(th + 40);
			const uint32_t constant_data_offset = k_type_header_offset + rd_u32(th + 44);
			const uint32_t clip_range_data_offset = k_type_header_offset + rd_u32(th + 48);

			if (num_tracks == 0)
			{
				d.num_segments = 0;
				d.image_size = image.reserve(0);
				return std::string();	// empty track list: seek/decompress are no-ops (decompression.transform.h:211-212)
			}
			if (num_segments == 0)
				return "clip without segments";
			for (int k = 0; k < 3; ++k)
				if (num_animated[k] > num_tracks || num_constant[k] > num_tracks)
					return "sub-track counts exceed the track count";

			const bool rot_variable = rotation_format == k_rot_drop_w_variable;
			const bool rot_full = rotation_format == k_rot_full;
			const bool variable[3] = { rot_variable, translation_format == 1, has_scale && scale_format == 1 };
			const uint32_t raw_marker = version >= k_version_raw31 ? 31u : 32u;		// animated_track_cache.transform.h:523
			const uint32_t segment_header_size = has_stripped ? 20u : 16u;				// compressed_headers.h:171-197
			const uint32_t num_entries = (num_tracks + 15) / 16;
			const uint32_t padded_rotations = align_up(num_animated[0], 4);
			const uint32_t num_animated_total = num_animated[0] + num_animated[1] + num_animated[2];
			const uint32_t num_kinds = has_scale ? 3u : 2u;

			// the per segment format / range tables are indexed by sub-track: the header's count must cover every variable sub-track
			// (compress.transform.impl.h:435 stores exactly this sum, rotations padded to groups of 4)
			{
				const uint64_t expected_variable = uint64_t(variable[0] ? padded_rotations : 0u) + (variable[1] ? num_animated[1] : 0u) + (variable[2] ? num_animated[2] : 0u);
				if (expected_variable > num_variable)
					return "num_animated_variable_sub_tracks is smaller than the variable sub-track counts";
			}
			if (!in_bounds(segment_headers_offset, uint64_t(segment_header_size) * num_segments))
				return "segment headers out of bounds";
			if (!in_bounds(sub_track_types_offset, uint64_t(num_entries) * 4 * num_kinds))
				return "sub-track types out of bounds";
			if (num_segments > 1 && !in_bounds(84, uint64_t(num_segments + 1) * 4))
				return "segment start indices out of bounds";

			d.flags |= has_scale ? k_clip_has_scale : 0u;
			d.flags |= ((misc >> 1) & 1) ? k_clip_default_scale_one : 0u;
			d.flags |= variable[0] ? k_clip_rot_variable : 0u;
			d.flags |= variable[1] ? k_clip_trans_variable : 0u;
			d.flags |= variable[2] ? k_clip_scale_variable : 0u;
			d.flags |= rot_full ? k_clip_rot_full : 0u;
			d.flags |= has_stripped ? k_clip_stripped : 0u;
			d.flags |= num_segments > 1 ? k_clip_has_segments : 0u;
			d.num_segments = num_segments;
			d.samples_per_segment = num_samples / num_segments;
			for (int k = 0; k < 3; ++k)
			{
				d.num_animated[k] = num_animated[k];
				d.num_constant[k] = num_constant[k];
			}
			d.num_animated_total = num_animated_total;

			// constant_track_cache_v0::initialize, constant_track_cache.transform.h:96-110
			const uint32_t constant_offset[3] = { constant_data_offset, constant_data_offset + (rot_full ? 16u : 12u) * num_constant[0],
				constant_data_offset + (rot_full ? 16u : 12u) * num_constant[0] + 12u * num_constant[1] };
			if (!in_bounds(constant_offset[2], 12ull * num_constant[2]))
				return "constant track data out of bounds";

			// animated_track_cache_v0::initialize, animated_track_cache.transform.h:1259-1262,1293-1294
			const uint32_t clip_range_offset[3] = { clip_range_data_offset, clip_range_data_offset + (variable[0] ? 24u * num_animated[0] : 0u),
				clip_range_data_offset + (variable[0] ? 24u * num_animated[0] : 0u) + (variable[1] ? 24u * num_animated[1] : 0u) };
			if ((variable[0] || variable[1] || variable[2]) && !in_bounds(clip_range_offset[2], variable[2] ? 24ull * num_animated[2] : 0ull))
				return "clip range data out of bounds";

			// ---- BoneDesc + the bone each animated sub-track belongs to ----
			d.bone_table_offset = image.reserve(size_t(num_tracks) * 8);
			std::vector<uint32_t> animated_bone[3];
			{
				uint32_t constant_rank[3] = { 0, 0, 0 };
				for (uint32_t kind = 0; kind < num_kinds; ++kind)
					animated_bone[kind].reserve(num_animated[kind]);
				for (uint32_t track = 0; track < num_tracks; ++track)
				{
					uint64_t desc = 0;
					for (uint32_t kind = 0; kind < num_kinds; ++kind)
					{
						// packed_sub_track_types: 16 sub-tracks per u32, 2 bits each, MSB first (compressed_headers.h:214-224)
						const uint32_t packed = rd_u32(blob + sub_track_types_offset + 4 * (kind * num_entries + track / 16));
						const uint32_t type = (packed >> ((15 - track % 16) * 2)) & 3;
						if (type == 3)
							return "invalid sub-track type";
						uint32_t rank = 0;
						if (type == 1)
							rank = constant_rank[kind]++;
						else if (type == 2)
						{
							rank = uint32_t(animated_bone[kind].size());
							animated_bone[kind].push_back(track);
						}
						desc |= (uint64_t(type) | (uint64_t(rank) << 2)) << (k_bone_kind_shift * kind);
					}
					std::memcpy(image.at(d.bone_table_offset) + size_t(track) * 8, &desc, 8);
				}
				for (uint32_t kind = 0; kind < num_kinds; ++kind)
					if (constant_rank[kind] != num_constant[kind] || animated_bone[kind].size() != num_animated[kind])
						return "sub-track types disagree with the header counts";
			}

			// ---- constant rotations: W reconstruction (and normalisation) done once, with the decoder's own operations ----
			d.const_rot_offset = image.reserve(size_t(num_constant[0]) * 32);
			for (uint32_t index = 0; index < num_constant[0]; ++index)
			{
				float q[4];
				if (rot_full)
				{
					for (int c = 0; c < 4; ++c)
						q[c] = rd_f32(blob + constant_offset[0] + index * 16 + c * 4);
				}
				else
				{
					// SOA groups of 4 with an unpadded last group (constant_track_cache.transform.h:153-170)
					const uint32_t group = index / 4, lane = index % 4;
					const uint32_t remaining = num_constant[0] - group * 4;
					const uint32_t group_size = remaining < 4 ? remaining : 4;
					const uint8_t* p = blob + constant_offset[0] + group * 48 + lane * 4;
					q[0] = rd_f32(p + group_size * 4 * 0);
					q[1] = rd_f32(p + group_size * 4 * 1);
					q[2] = rd_f32(p + group_size * 4 * 2);
					// quat_from_positive_w4, math/quatf.h:135-147
					float r = 1.0F - q[0] * q[0];
					r = r - q[1] * q[1];
					r = r - q[2] * q[2];
					q[3] = std::sqrt(std::fabs(r));
				}
				float n[4] = { q[0], q[1], q[2], q[3] };
				if (!rot_full)
				{
					// quat_normalize4, math/quatf.h:200-211 (policy `always`, constant_track_cache.transform.h:172-175)
					float dot = n[0] * n[0];
					dot = n[1] * n[1] + dot;
					dot = n[2] * n[2] + dot;
					dot = n[3] * n[3] + dot;
					const float inv_len = 1.0F / std::sqrt(dot);
					for (int c = 0; c < 4; ++c)
						n[c] = n[c] * inv_len;
				}
				std::memcpy(image.at(d.const_rot_offset) + size_t(index) * 32, q, 16);
				std::memcpy(image.at(d.const_rot_offset) + size_t(index) * 32 + 16, n, 16);
			}

			// ---- constant translations then scales, one float4 each ----
			d.const_vec_offset = image.reserve(size_t(num_constant[1] + num_constant[2]) * 16);
			for (uint32_t kind = 1; kind <= 2; ++kind)
				for (uint32_t index = 0; index < num_constant[kind]; ++index)
				{
					const size_t slot = (kind == 2 ? num_constant[1] : 0u) + index;
					std::memcpy(image.at(d.const_vec_offset) + slot * 16, blob + constant_offset[kind] + index * 12, 12);
				}

			// ---- AnimDesc: clip range + destination bone of every animated sub-track ----
			d.anim_table_offset = image.reserve(size_t(num_animated_total) * sizeof(AnimDesc));
			{
				uint32_t slot = 0;
				for (uint32_t kind = 0; kind < 3; ++kind)
					for (uint32_t index = 0; index < num_animated[kind]; ++index, ++slot)
					{
						AnimDesc anim = {};
						anim.bone = animated_bone[kind][index];
						anim.extent[0] = anim.extent[1] = anim.extent[2] = 1.0F;
						if (variable[kind])
						{
							if (kind == 0)
							{
								// remap_clip_range_data4, animated_track_cache.transform.h:391-418: SOA per group of 4, last group unpadded
								const uint32_t group = index / 4, lane = index % 4;
								const uint32_t remaining = num_animated[0] - group * 4;
								const uint32_t group_size = remaining < 4 ? remaining : 4;
								const uint8_t* p = blob + clip_range_offset[0] + group * 96 + lane * 4;
								for (int c = 0; c < 3; ++c)
								{
									anim.min[c] = rd_f32(p + group_size * 4 * c);
									anim.extent[c] = rd_f32(p + group_size * 4 * (3 + c));
								}
							}
							else
							{
								// unpack_animated_vector3, :949-958: min xyz then extent xyz
								const uint8_t* p = blob + clip_range_offset[kind] + index * 24;
								for (int c = 0; c < 3; ++c)
								{
									anim.min[c] = rd_f32(p + 4 * c);
									anim.extent[c] = rd_f32(p + 12 + 4 * c);
								}
							}
						}
						// stored as two arrays of 16 byte halves (layout.h): a warp's loads of consecutive sub-tracks are then contiguous
						std::memcpy(image.at(d.anim_table_offset) + size_t(slot) * 16, &anim, 16);
						std::memcpy(image.at(d.anim_table_offset) + (size_t(num_animated_total) + slot) * 16, reinterpret_cast<const uint8_t*>(&anim) + 16, 16);
					}
			}

			// ---- segment start indices (+ sentinel), transform_tracks_header::get_segment_start_indices, compressed_headers.h:271-272 ----
			if (num_segments > 1)
			{
				d.start_indices_offset = image.reserve(size_t(num_segments + 1) * 4);
				std::memcpy(image.at(d.start_indices_offset), blob + 84, size_t(num_segments + 1) * 4);
			}

			// ---- per segment: SegDesc, entries, stream ----
			d.seg_table_offset = image.reserve(size_t(num_segments) * sizeof(SegDesc));
			for (uint32_t segment = 0; segment < num_segments; ++segment)
			{
				const uint8_t* header = blob + segment_headers_offset + segment_header_size * segment;
				const uint32_t pose_bit_size = rd_u32(header + 0);
				const uint32_t rotation_bit_size = rd_u32(header + 4);
				const uint32_t translation_bit_size = rd_u32(header + 8);
				const uint32_t segment_data = k_type_header_offset + rd_u32(header + 12);

				// transform_tracks_header::get_segment_data, compressed_headers.h:310-324 (the blob is 16 byte aligned, so aligning
				// offsets equals aligning addresses)
				const uint32_t format_offset = segment_data;
				const uint32_t range_offset = align_up(format_offset + num_variable, 2);
				const uint32_t range_size = num_segments > 1 ? 6u * num_variable : 0u;
				const uint32_t animated_offset = align_up(range_offset + range_size, 4);
				if (!in_bounds(format_offset, num_variable) || !in_bounds(range_offset, range_size) || !in_bounds(animated_offset, 0))
					return "segment data out of bounds";

				SegDesc seg = {};
				seg.pose_bit_size = pose_bit_size;
				seg.sample_indices = has_stripped ? rd_u32(header + 16) : 0xFFFFFFFFu;
				seg.blob_format_offset = format_offset;
				seg.blob_range_offset = range_offset;
				seg.blob_animated_offset = animated_offset;

				// Number of stored key frames (stripped segments store popcount(sample_indices) frames)
				uint32_t stored_key_frames;
				if (has_stripped)
					stored_key_frames = uint32_t(__builtin_popcount(seg.sample_indices));
				else if (num_segments == 1)
					stored_key_frames = num_samples;
				else
				{
					const uint32_t start = rd_u32(blob + 84 + 4 * segment);
					const uint32_t next = segment + 1 < num_segments ? rd_u32(blob + 84 + 4 * (segment + 1)) : num_samples;
					if (next < start)
						return "segment start indices are not sorted";
					stored_key_frames = next - start;
				}
				const uint64_t stream_bytes = (uint64_t(pose_bit_size) * stored_key_frames + 7) / 8;
				if (!in_bounds(animated_offset, stream_bytes) || stream_bytes > 0xFFFFFF00ull)
					return "animated data out of bounds";
				seg.stream_bytes = uint32_t(stream_bytes);
				if (has_database)
					out.db_pose_bits.push_back(pose_bit_size);
				const uint32_t key_frame_bytes = (pose_bit_size + 7) / 8;
				out.max_key_frame_bytes = key_frame_bytes > out.max_key_frame_bytes ? key_frame_bytes : out.max_key_frame_bytes;

				// Entries. Bit offsets are the running sum of segment_animated_sampling_context_v0::animated_track_data_bit_offset
				// (animated_track_cache.transform.h:598-599,653; cursors set up at :1240-1308). Rotation metadata and segment range
				// data are padded to groups of 4, translations / scales are not (:1264-1276,1296-1302).
				seg.entries_offset = image.reserve(size_t(num_animated_total) * sizeof(Entry));
				const uint8_t* format = blob + format_offset;
				const uint8_t* range = blob + range_offset;
				const uint32_t kind_bit_offset[3] = { 0u, rotation_bit_size, rotation_bit_size + translation_bit_size };
				const uint32_t kind_format_offset[3] = { 0u, variable[0] ? padded_rotations : 0u,
					(variable[0] ? padded_rotations : 0u) + (variable[1] ? num_animated[1] : 0u) };
				uint32_t slot = 0;
				for (uint32_t kind = 0; kind < 3; ++kind)
				{
					uint32_t bit_offset = kind_bit_offset[kind];
					for (uint32_t index = 0; index < num_animated[kind]; ++index, ++slot)
					{
						Entry entry = {};
						uint32_t code, stream_bits;
						entry.inv_max = 1.0F;
						if (variable[kind])
						{
							const uint32_t stored = format[kind_format_offset[kind] + index];
							// the 6 segment range bytes of this sub-track: min xyz, extent xyz
							uint8_t r[6] = { 0, 0, 0, 0, 0, 0 };
							if (num_segments > 1)
							{
								if (kind == 0)
								{
									// SOA per group of 4: min.xxxx min.yyyy min.zzzz extent.xxxx extent.yyyy extent.zzzz (:159)
									const uint8_t* p = range + (index / 4) * 24 + (index % 4);
									for (int c = 0; c < 6; ++c)
										r[c] = p[4 * c];
								}
								else
									std::memcpy(r, range + kind_format_offset[kind] * 6 + index * 6, 6);	// AOS (:936-940)
							}
							if (stored == 0)
							{
								// constant inside the segment, 16 bits per component (:552-587 rotations, unpack_vector3_u48_unsafe for vectors)
								if (num_segments == 1)
									return "constant bit rate inside a single segment clip";
								uint32_t x, y, z;
								if (kind == 0)
								{
									x = (uint32_t(r[0]) << 8) | r[1];
									y = (uint32_t(r[2]) << 8) | r[3];
									z = (uint32_t(r[4]) << 8) | r[5];
								}
								else
								{
									x = uint32_t(r[0]) | (uint32_t(r[1]) << 8);
									y = uint32_t(r[2]) | (uint32_t(r[3]) << 8);
									z = uint32_t(r[4]) | (uint32_t(r[5]) << 8);
								}
								code = 0;
								stream_bits = 0;
								entry.range_lo = x | (y << 16);
								entry.range_hi = z;
								entry.inv_max = 1.0F / 65535.0F;
							}
							else if (stored == raw_marker)
							{
								code = 32u | k_entry_raw;
								stream_bits = 96;
							}
							else if (stored <= 23)
							{
								code = stored;
								stream_bits = stored * 3;
								// the bytes unpack_segment_range_data reads (:157-298; vectors math/vector4_packing.h:781-818), expanded by the kernels
								entry.range_lo = uint32_t(r[0]) | (uint32_t(r[1]) << 8) | (uint32_t(r[2]) << 16) | (uint32_t(r[3]) << 24);
								entry.range_hi = uint32_t(r[4]) | (uint32_t(r[5]) << 8);
								entry.inv_max = inv_max_value(stored);
							}
							else
								return "invalid per track bit count";
						}
						else
						{
							code = 32u | k_entry_raw;
							stream_bits = (kind == 0 && rot_full) ? 128u : 96u;
						}
						if (bit_offset >= (1u << 24))
							return "key frame too large for the sub-track entry table";
						entry.offset_code = (bit_offset << 8) | code;
						std::memcpy(image.at(seg.entries_offset) + size_t(slot) * sizeof(Entry), &entry, sizeof(Entry));
						bit_offset += stream_bits;
					}
					if (bit_offset > pose_bit_size && num_animated[kind] != 0)
						return "sub-track bit widths exceed the animated pose size";
				}

				seg.stream_offset = append_stream(image, blob + animated_offset, size_t(stream_bytes));
				std::memcpy(image.at(d.seg_table_offset) + size_t(segment) * sizeof(SegDesc), &seg, sizeof(seg));
			}

			d.image_size = image.reserve(0);
			return std::string();
		}
	}

	aclb200_status set_error(aclb200_context* context, aclb200_status status, const std::string& message)
	{
		if (context != nullptr)
			context->last_error = message;
		return status;
	}

	aclb200_status check_cuda(aclb200_context* context, cudaError_t error, const char* what)
	{
		if (error == cudaSuccess)
			return ACLB200_OK;
		const aclb200_status status = error == cudaErrorMemoryAllocation ? ACLB200_ERR_OUT_OF_MEMORY : ACLB200_ERR_CUDA;
		return set_error(context, status, std::string(what) + ": " + cudaGetErrorString(error));
	}

	namespace
	{
		// host threads the transcode may use: the scheduler affinity of the calling thread, at most 32
		uint32_t transcode_threads(uint32_t num_clips)
		{
			uint32_t threads = std::thread::hardware_concurrency();
#if defined(__linux__)
			cpu_set_t set;
			if (sched_getaffinity(0, sizeof(set), &set) == 0)
				threads = uint32_t(CPU_COUNT(&set));
#endif
			if (threads > 32) threads = 32;
			if (threads > num_clips / 64) threads = num_clips / 64;		// not worth a thread for a handful of clips
			return threads == 0 ? 1 : threads;
		}

		// runs job(thread_index, first, last) over [0, count) split into contiguous ranges, on `threads` threads
		template<class Job>
		void parallel_ranges(uint32_t count, uint32_t threads, const Job& job)
		{
			if (threads <= 1)
			{
				job(0u, 0u, count);
				return;
			}
			std::vector<std::thread> pool;
			pool.reserve(threads);
			for (uint32_t t = 0; t < threads; ++t)
				pool.emplace_back([&, t]() { job(t, uint32_t(uint64_t(count) * t / threads), uint32_t(uint64_t(count) * (t + 1) / threads)); });
			for (std::thread& thread : pool)
				thread.join();
		}
	}

	aclb200_status build_clipset(aclb200_context* context, const std::function<const uint8_t*(uint32_t)>& get_blob, const uint32_t* sizes,
		uint32_t num_clips, bool check_hash, aclb200_clipset** out_clipset, uint32_t* out_failed_clip)
	{
		if (context == nullptr || out_clipset == nullptr || sizes == nullptr || num_clips == 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "upload_clips: null argument or empty clip list");
		*out_clipset = nullptr;

		aclb200_clipset* set = nullptr;
		try
		{
			set = new aclb200_clipset();
			set->device = context->device;
			set->host_clips.resize(num_clips);
			set->host_looping.resize(num_clips);
			set->host_blob_db_offset.resize(num_clips);
			set->host_db_pose_bits.resize(num_clips);

			auto fail = [&](aclb200_status status, const std::string& message, uint32_t clip)
			{
				if (out_failed_clip != nullptr)
					*out_failed_clip = clip;
				delete set;
				return set_error(context, status, message);
			};

			// Pass 1 (host threads, clips split into contiguous ranges): validate every clip and measure its image. Nothing is kept but
			// the descriptors: a multi-GB clip set never needs a second full host copy.
			const uint32_t threads = transcode_threads(num_clips);
			struct range_result
			{
				uint32_t failed_clip = 0xFFFFFFFFu;
				bool unsupported = false;
				std::string error;
				uint32_t max_key_frame_bytes = 0;
			};
			std::vector<range_result> results(threads);
			std::vector<uint32_t> track_types(num_clips);
			parallel_ranges(num_clips, threads, [&](uint32_t t, uint32_t first, uint32_t last)
			{
				std::vector<uint8_t> staging;
				parse_result parsed;
				range_result& result = results[t];
				for (uint32_t clip = first; clip < last; ++clip)
				{
					bool unsupported = false;
					staging.clear();
					std::string error;
					try
					{
						error = transcode_clip(get_blob(clip), sizes[clip], check_hash, staging, parsed, unsupported);
					}
					catch (const image_too_large&)
					{
						error = "the clip image would pass 4 GiB";
						unsupported = true;
					}
					catch (const std::bad_alloc&)
					{
						error = "out of host memory";
						unsupported = true;
					}
					if (!error.empty())
					{
						result.failed_clip = clip;
						result.unsupported = unsupported;
						result.error = error;
						return;
					}
					set->host_clips[clip] = parsed.desc;
					set->host_looping[clip] = parsed.looping_policy;
					set->host_blob_db_offset[clip] = parsed.db_clip_header_offset;
					set->host_db_pose_bits[clip] = parsed.db_pose_bits;
					track_types[clip] = parsed.track_type;
					result.max_key_frame_bytes = parsed.max_key_frame_bytes > result.max_key_frame_bytes ? parsed.max_key_frame_bytes : result.max_key_frame_bytes;
				}
			});
			for (const range_result& result : results)		// ranges are in clip order: the first failure is the lowest clip
				if (result.failed_clip != 0xFFFFFFFFu)
					return fail(result.unsupported ? ACLB200_ERR_UNSUPPORTED : ACLB200_ERR_INVALID_CLIP,
						"clip " + std::to_string(result.failed_clip) + ": " + result.error, result.failed_clip);

			uint64_t blob_bytes = 0, total_image_bytes = 0;
			const uint32_t set_track_type = track_types[0];
			uint32_t max_tracks = 0, min_tracks = std::numeric_limits<uint32_t>::max();
			for (uint32_t clip = 0; clip < num_clips; ++clip)
			{
				if (track_types[clip] != set_track_type)
					return fail(ACLB200_ERR_UNSUPPORTED, "clip " + std::to_string(clip) + ": a clip set holds a single track type", clip);
				ClipDesc& desc = set->host_clips[clip];
				desc.data_offset = total_image_bytes;
				total_image_bytes += align_up64(desc.image_size, k_section_alignment);
				blob_bytes += desc.size;
				max_tracks = desc.num_tracks > max_tracks ? desc.num_tracks : max_tracks;
				if (desc.num_tracks % 2 != 0)
					set->all_tracks_even = false;
				min_tracks = desc.num_tracks < min_tracks ? desc.num_tracks : min_tracks;
				if (set_track_type == k_track_qvvf)
				{
					for (int k = 0; k < 3; ++k)
						set->max_animated[k] = desc.num_animated[k] > set->max_animated[k] ? desc.num_animated[k] : set->max_animated[k];
					set->max_animated_total = desc.num_animated_total > set->max_animated_total ? desc.num_animated_total : set->max_animated_total;
				}
			}
			for (const range_result& result : results)
					set->max_key_frame_bytes = result.max_key_frame_bytes > set->max_key_frame_bytes ? result.max_key_frame_bytes : set->max_key_frame_bytes;
			total_image_bytes += k_stream_tail;

			set->info.num_clips = num_clips;
			set->info.track_type = set_track_type;
			set->info.max_tracks = max_tracks;
			set->info.min_tracks = min_tracks;
			set->info.blob_bytes = blob_bytes;
			set->info.index_bytes = total_image_bytes;

			// Pass 2: device allocation, then chunk by chunk: the host threads transcode the chunk's clips straight to their final
			// offsets inside a staging buffer, one copy brings it to the device.
			cudaError_t error = cudaSetDevice(context->device);
			if (error == cudaSuccess) error = cudaMalloc(reinterpret_cast<void**>(&set->d_data), total_image_bytes);
			if (error == cudaSuccess) error = cudaMalloc(reinterpret_cast<void**>(&set->d_clips), sizeof(ClipDesc) * size_t(num_clips));
			if (error == cudaSuccess) error = cudaMemset(set->d_data + (total_image_bytes - k_stream_tail), 0, k_stream_tail);
			const uint64_t staging_capacity = uint64_t(256) << 20;
			std::vector<uint8_t> staging;
			for (uint32_t chunk_first = 0; chunk_first < num_clips && error == cudaSuccess; )
			{
				uint32_t chunk_last = chunk_first;
				const uint64_t chunk_base = set->host_clips[chunk_first].data_offset;
				uint64_t chunk_bytes = 0;
				while (chunk_last < num_clips && (chunk_last == chunk_first || chunk_bytes + align_up64(set->host_clips[chunk_last].image_size, k_section_alignment) <= staging_capacity))
				{
					chunk_bytes += align_up64(set->host_clips[chunk_last].image_size, k_section_alignment);
					++chunk_last;
				}
				staging.assign(size_t(chunk_bytes), 0);
				std::atomic<bool> out_of_memory(false);
				parallel_ranges(chunk_last - chunk_first, threads, [&](uint32_t, uint32_t first, uint32_t last)
				{
					try
					{
						std::vector<uint8_t> image;
						parse_result parsed;
						for (uint32_t clip = chunk_first + first; clip < chunk_first + last; ++clip)
						{
							bool unsupported = false;
							image.clear();
							transcode_clip(get_blob(clip), sizes[clip], false, image, parsed, unsupported);		// validated by pass 1
							std::memcpy(staging.data() + (set->host_clips[clip].data_offset - chunk_base), image.data(), image.size());
						}
					}
					catch (...)		// an exception may not leave a thread
					{
						out_of_memory.store(true);
					}
				});
				if (out_of_memory.load())
					throw std::bad_alloc();
				error = cudaMemcpy(set->d_data + chunk_base, staging.data(), size_t(chunk_bytes), cudaMemcpyHostToDevice);
				chunk_first = chunk_last;
			}
			if (error == cudaSuccess) error = cudaMemcpy(set->d_clips, set->host_clips.data(), sizeof(ClipDesc) * size_t(num_clips), cudaMemcpyHostToDevice);
			if (error != cudaSuccess)
			{
				const aclb200_status status = check_cuda(context, error, "upload_clips");
				cudaFree(set->d_data);
				cudaFree(set->d_clips);
				delete set;
				return status;
			}

			*out_clipset = set;
			return ACLB200_OK;
		}
		catch (const std::exception&)
		{
			// (std::bad_alloc, std::system_error of a thread that could not start) nothing may unwind through the extern "C" boundary
			if (set != nullptr)
			{
				cudaFree(set->d_data);
				cudaFree(set->d_clips);
				delete set;
			}
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "upload_clips: out of host memory");
		}
	}
}
