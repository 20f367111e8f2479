// acl_b200/csrc/layout.h -- what lives in HBM for a clip set, shared by the host builder (clipset.cpp) and the kernels.
//
// At upload every compressed_tracks blob is TRANSCODED once into a GPU-native "clip image"; the original bytes are not
// kept on the device. The compressed payload itself (the variable bit rate key frame streams) is carried over bit for
// bit -- only the byte order inside each 32-bit word is normalised so a little-endian machine can read the big-endian
// stream with aligned word loads -- while the metadata the CPU decoder walks with serial cursors is re-laid out so that
// every (request, sub-track) is independent work and needs one or two 16-byte loads:
//
//   clips : ClipDesc[num_clips]                   what decompression_context::initialize() caches (initialize_v0,
//                                                 includes/acl/decompression/impl/decompression.transform.h:84-132)
//   data  : per clip, 16-byte aligned sections
//     BoneDesc[num_tracks]            u64   (type, rank) of the rotation / translation / scale sub-track of each bone: the
//                                           prefix popcounts of decompress_track_v0 (decompression.transform.h:1873-1891)
//     ConstRot[num_constant_rot][2]   f32x4 constant rotations with W already reconstructed (quat_from_positive_w4,
//                                           math/quatf.h:135-147), [1] = also normalised (policy `always`); same IEEE ops on the host
//     ConstVec[num_constant_trans + num_constant_scale] f32x4 constant translations then scales
//     AnimDesc[num_animated_total]    48 B  clip range of each animated sub-track (remap_clip_range_data4 /
//                                           unpack_animated_vector3, animated_track_cache.transform.h:391-466,947-958) + the bone
//                                           it belongs to (the "select" the CPU does by walking the 2-bit type arrays)
//     start_indices[num_segments + 1] u32   segment_start_indices + sentinel (only when num_segments > 1)
//     SegDesc[num_segments]           32 B
//     Entry[num_segments][num_animated_total] 16 B  per segment and sub-track: bit offset inside a key frame (the running sum of
//                                           animated_track_data_bit_offset, animated_track_cache.transform.h:598-599,653), bit
//                                           width, 1 / (2^bits - 1) and the six segment range bytes as stored (or the constant
//                                           sample when the bit rate is 0)
//     stream[num_segments]            u32[] key frames of the segment, byte-swapped words, 16-byte aligned, 64 B zero tail
#pragma once

#include <stdint.h>

namespace aclb200
{
	// ---- reference binary format constants (includes/acl/core/impl/compressed_headers.h) ----------------
	constexpr uint32_t k_tag = 0xac11ac11u;						// core/buffer_tag.h:49
	constexpr uint32_t k_version_first = 7;						// v02_00_00, core/compressed_tracks_version.h:75
	constexpr uint32_t k_version_raw31 = 9;						// v02_01_99_1: raw bit rate stored as 31 in the per-track format
	constexpr uint32_t k_version_latest = 10;					// v02_01_00
	constexpr uint32_t k_track_qvvf = 12;						// core/track_types.h:68
	constexpr uint32_t k_type_header_offset = 32;				// transform_tracks_header / scalar_tracks_header
	constexpr uint32_t k_transform_header_size = 52;
	constexpr uint32_t k_section_alignment = 16;
	constexpr uint32_t k_stream_tail = 64;						// zero bytes after every stream (the reference pads 15, compress.transform.impl.h:395-396)

	constexpr uint32_t k_rot_full = 0;							// rotation_format8, core/track_formats.h:48-53
	constexpr uint32_t k_rot_drop_w_full = 2;
	constexpr uint32_t k_rot_drop_w_variable = 3;

	// ---- ClipDesc::flags ---------------------------------------------------------------------------------
	constexpr uint32_t k_clip_has_scale = 1u << 0;
	constexpr uint32_t k_clip_default_scale_one = 1u << 1;
	constexpr uint32_t k_clip_rot_variable = 1u << 2;
	constexpr uint32_t k_clip_trans_variable = 1u << 3;
	constexpr uint32_t k_clip_scale_variable = 1u << 4;
	constexpr uint32_t k_clip_rot_full = 1u << 5;				// quatf_full: 4 stored components, no W reconstruction
	constexpr uint32_t k_clip_stripped = 1u << 6;				// has_stripped_keyframes
	constexpr uint32_t k_clip_wrap = 1u << 7;					// compressed_tracks::get_looping_policy() == wrap
	constexpr uint32_t k_clip_has_segments = 1u << 8;			// more than one segment => segment range data exists

	struct alignas(16) ClipDesc
	{
		uint64_t data_offset;				// byte offset of the clip image inside the data buffer
		uint32_t num_tracks;
		uint32_t num_samples;
		float    sample_rate;
		uint32_t flags;
		uint32_t num_segments;
		uint32_t samples_per_segment;		// num_samples / num_segments (the reference's segment guess, decompression.transform.h:377)
		float    duration_clamp;			// get_finite_duration(clamp), core/impl/compressed_tracks.impl.h:113-134
		float    duration_wrap;				// get_finite_duration(wrap)
		uint32_t num_animated[3];			// rotation, translation, scale
		uint32_t num_constant[3];
		// image relative byte offsets
		uint32_t bone_table_offset;			// BoneDesc[num_tracks]            (scalar clips: ScalarTrackDesc[num_tracks])
		uint32_t const_rot_offset;			// float4[num_constant[0]][2]      (scalar clips: constant values)
		uint32_t const_vec_offset;			// float4[num_constant[1] + [2]]   (scalar clips: range values)
		uint32_t anim_table_offset;			// AnimDesc[num_animated_total]
		uint32_t start_indices_offset;		// u32[num_segments + 1]
		uint32_t seg_table_offset;			// SegDesc[num_segments]           (scalar clips: offset of the single stream)
		uint32_t num_animated_total;		// (scalar clips: num_bits_per_frame)
		uint32_t image_size;
		uint32_t hash;						// compressed_tracks::get_hash()
		uint32_t size;						// compressed_tracks::get_size()
		uint32_t track_range_offset;		// scalar clips: float[num_tracks][2 * components] = range min, range extent of every track (constant
											// tracks: the constant, 0; raw tracks: 0, 1), so that a thread finds them without the descriptor's index
		uint32_t pad;
	};
	static_assert(sizeof(ClipDesc) % 16 == 0, "ClipDesc must stay 16 byte sized");

	// BoneDesc: one u64 per bone. kind k in {0 rotation, 1 translation, 2 scale}:
	//   type  = (desc >> (22 * k)) & 3          0 default, 1 constant, 2 animated (packed_sub_track_types, compressed_headers.h:214-224)
	//   index = (desc >> (22 * k + 2)) & 0xFFFFF rank among the constant or animated sub-tracks of that kind
	constexpr uint32_t k_bone_kind_shift = 22;
	constexpr uint32_t k_bone_index_mask = 0xFFFFFu;
	constexpr uint32_t k_max_tracks = 1u << 18;					// the scale rank has 18 bits left

	// Clip-level data of one animated sub-track: two 16 byte loads give the clip range and the destination bone.
	// In the image the table is stored as two arrays, first16[num_animated_total] then second16[num_animated_total]:
	// the threads of a warp handle consecutive sub-tracks, so each of their 16 byte loads covers one contiguous 512 byte run
	// (4 L1 wavefronts) instead of every other 16 bytes of a 1 KB run (8 wavefronts) -- the L1 data pipe is this kernel's busiest unit.
	struct alignas(16) AnimDesc
	{
		float    extent[3];		// clip range extent xyz (1.0 when the format carries no clip range)
		uint32_t bone;			// track index this sub-track writes to
		float    min[3];		// clip range min xyz (0.0 when the format carries no clip range)
		uint32_t pad;
	};
	static_assert(sizeof(AnimDesc) == 32, "AnimDesc is 32 bytes");

	struct alignas(16) SegDesc
	{
		uint32_t stream_offset;				// image relative, 16 byte aligned: byte-swapped 32-bit words of the segment's key frames
		uint32_t pose_bit_size;				// segment_header::animated_pose_bit_size
		uint32_t sample_indices;			// stripped_segment_header_t::sample_indices (0xFFFFFFFF when nothing is stripped)
		uint32_t entries_offset;			// image relative: Entry[num_animated_total]
		// offsets inside the ORIGINAL blob, reported by the seek parity hook (persistent_transform_decompression_context_v0)
		uint32_t blob_format_offset;
		uint32_t blob_range_offset;
		uint32_t blob_animated_offset;
		uint32_t stream_bytes;				// bytes of key frame data stored (without the tail)
	};
	static_assert(sizeof(SegDesc) == 32, "SegDesc is 32 bytes");

	// Entry::offset_code = (bit offset inside the key frame << 8) | code
	//   code 1..23           bits per component, quantised, segment + clip range apply
	//   code 0               constant inside the segment: the range bytes hold the 3 x 16 bit sample, only the clip range applies
	//   code 32 | k_entry_raw  raw 32-bit floats (3 components, 4 for quatf_full rotations), no range applies
	constexpr uint32_t k_entry_raw = 0x80u;
	struct alignas(16) Entry
	{
		uint32_t offset_code;
		float    inv_max;		// 1 / (2^code - 1) (PackedTableEntry::max_value, math/vector4_packing.h:927-929); 1 / 65535 for code 0
		// code 1..23: the six segment range bytes of the sub-track as the clip stores them, min x, y, z then extent x, y, z (byte 0 of
		// range_lo is min x, byte 1 of range_hi is extent z); the kernels expand a byte as u8 * (1 / 255) in float, the one IEEE
		// multiply of unpack_segment_range_data (animated_track_cache.transform.h:157-298).
		// code 0: the three 16 bit integers of the constant sample, x | y << 16 in range_lo and z in range_hi.
		// raw: zero (the decoders use min = 0, extent = 1: an ignored range still multiplies by 1 and adds 0).
		// One 16 byte load per entry: the threads of a warp read consecutive entries, one contiguous 512 byte run.
		uint32_t range_lo;
		uint32_t range_hi;
	};
	static_assert(sizeof(Entry) == 16, "Entry is 16 bytes");

	// Scalar clips (decompression/impl/decompression.scalar.h): one descriptor per track.
	struct alignas(16) ScalarTrackDesc
	{
		uint32_t bit_offset;			// inside a frame
		uint32_t value_index_and_bits;	// (index of the first float in constant / range values << 8) | num_bits (0 constant, 32 raw)
		float    inv_max;
		uint32_t pad;
	};
}
