// oracle/ref_root_motion.cpp -- TEST INFRASTRUCTURE ONLY: root motion from the unmodified reference, compiled into
// _ref/libaclref_root_motion.so (oracle/root_motion.mk) with the flags of the reference build where the reference tree exists.
//   - rtm::qvv_inverse / rtm::qvv_mul on given rows, and the composition of aclb200_extract_root_motion on given root samples;
//   - the whole path: acl::decompression_context, set_looping_policy(clamp), seek and decompress_tracks with a track_writer that keeps the
//     root's row only, at from_time, to_time and the clip's two ends, then the composition.
// Rows are 12 floats (rotation xyzw, translation xyz + w, scale xyz + w); the rows written carry 0 in both w lanes.
#include <acl/core/compressed_tracks.h>
#include <acl/core/track_writer.h>
#include <acl/decompression/decompress.h>
#include <rtm/qvvf.h>

#include <cstddef>
#include <cstdint>
#include <cstring>

namespace
{
	using namespace acl;

	// the settings kinds of oracle/ref_tool.cpp (decompression_settings.h:74-232)
	struct settings_benchmark final : public default_transform_decompression_settings
	{
		static constexpr compressed_tracks_version16 version_supported() { return compressed_tracks_version16::latest; }
		static constexpr bool skip_initialize_safety_checks() { return true; }
	};
	struct settings_never final : public debug_transform_decompression_settings
	{
		static constexpr rotation_normalization_policy_t get_rotation_normalization_policy() { return rotation_normalization_policy_t::never; }
		static constexpr bool is_per_track_rounding_supported() { return false; }
	};
	struct settings_all_lerp final : public debug_transform_decompression_settings
	{
		static constexpr rotation_normalization_policy_t get_rotation_normalization_policy() { return rotation_normalization_policy_t::lerp_only; }
		static constexpr bool is_per_track_rounding_supported() { return false; }
	};
	struct settings_raw_only final : public decompression_settings
	{
		static constexpr bool is_track_type_supported(track_type8 type) { return type == track_type8::qvvf; }
		static constexpr bool is_rotation_format_supported(rotation_format8 format) { return format == rotation_format8::quatf_full; }
		static constexpr bool is_translation_format_supported(vector_format8 format) { return format == vector_format8::vector3f_full; }
		static constexpr bool is_scale_format_supported(vector_format8 format) { return format == vector_format8::vector3f_full; }
		static constexpr bool is_per_track_rounding_supported() { return false; }
	};

	// A track_writer (core/track_writer.h:82-216) that keeps the root track's row and drops every other track's
	struct root_writer_base : public track_writer
	{
		uint32_t root = 0;
		float* row = nullptr;
		const uint8_t* per_track_rounding = nullptr;
		const float* variable_defaults = nullptr;
		float constant_defaults[12] = { 0, 0, 0, 1,  0, 0, 0, 0,  1, 1, 1, 0 };

		sample_rounding_policy get_rounding_policy(sample_rounding_policy seek_policy, uint32_t track_index) const
		{
			if (seek_policy != sample_rounding_policy::per_track || per_track_rounding == nullptr)
				return seek_policy;
			return static_cast<sample_rounding_policy>(per_track_rounding[track_index]);
		}

		rtm::quatf RTM_SIMD_CALL get_constant_default_rotation() const { return rtm::quat_load(&constant_defaults[0]); }
		rtm::vector4f RTM_SIMD_CALL get_constant_default_translation() const { return rtm::vector_load(&constant_defaults[4]); }
		rtm::vector4f RTM_SIMD_CALL get_constant_default_scale() const { return rtm::vector_load(&constant_defaults[8]); }
		rtm::quatf RTM_SIMD_CALL get_variable_default_rotation(uint32_t track_index) const { return rtm::quat_load(&variable_defaults[track_index * 12 + 0]); }
		rtm::vector4f RTM_SIMD_CALL get_variable_default_translation(uint32_t track_index) const { return rtm::vector_load(&variable_defaults[track_index * 12 + 4]); }
		rtm::vector4f RTM_SIMD_CALL get_variable_default_scale(uint32_t track_index) const { return rtm::vector_load(&variable_defaults[track_index * 12 + 8]); }

		void RTM_SIMD_CALL write_rotation(uint32_t track_index, rtm::quatf_arg0 rotation) { if (track_index == root) rtm::quat_store(rotation, &row[0]); }
		void RTM_SIMD_CALL write_translation(uint32_t track_index, rtm::vector4f_arg0 translation) { if (track_index == root) rtm::vector_store3(translation, &row[4]); }
		void RTM_SIMD_CALL write_scale(uint32_t track_index, rtm::vector4f_arg0 scale) { if (track_index == root) rtm::vector_store3(scale, &row[8]); }
	};

	// writer mode 0: the library defaults; 2: constant defaults from the writer; 3: per track defaults from the writer
	struct root_writer_legacy final : public root_writer_base {};
	struct root_writer_constant final : public root_writer_base
	{
		static constexpr default_sub_track_mode get_default_rotation_mode() { return default_sub_track_mode::constant; }
		static constexpr default_sub_track_mode get_default_translation_mode() { return default_sub_track_mode::constant; }
		static constexpr default_sub_track_mode get_default_scale_mode() { return default_sub_track_mode::constant; }
	};
	struct root_writer_variable final : public root_writer_base
	{
		static constexpr default_sub_track_mode get_default_rotation_mode() { return default_sub_track_mode::variable; }
		static constexpr default_sub_track_mode get_default_translation_mode() { return default_sub_track_mode::variable; }
		static constexpr default_sub_track_mode get_default_scale_mode() { return default_sub_track_mode::variable; }
	};

	rtm::qvvf load_row(const float* row)
	{
		return rtm::qvv_set(rtm::quat_load(row), rtm::vector_load(row + 4), rtm::vector_load(row + 8));
	}

	void store_row(const rtm::qvvf& q, float* row)
	{
		rtm::quat_store(q.rotation, row);
		rtm::vector_store3(q.translation, row + 4);
		rtm::vector_store3(q.scale, row + 8);
		row[7] = 0.0f;
		row[11] = 0.0f;
	}

	// rel(a, b) = qvv_mul(T(b), qvv_inverse(T(a)))
	rtm::qvvf relative(const rtm::qvvf& a, const rtm::qvvf& b)
	{
		return rtm::qvv_mul(b, rtm::qvv_inverse(a));
	}

	rtm::qvvf compose(const rtm::qvvf& from, const rtm::qvvf& to, const rtm::qvvf& end, const rtm::qvvf& start, int32_t cycles)
	{
		if (cycles == 0)
			return relative(from, to);
		const rtm::qvvf& reached = cycles > 0 ? end : start;
		const rtm::qvvf& resumed = cycles > 0 ? start : end;
		rtm::qvvf motion = relative(from, reached);
		const rtm::qvvf cycle = relative(resumed, reached);
		for (int32_t i = 1; i < (cycles > 0 ? cycles : -cycles); ++i)
			motion = rtm::qvv_mul(cycle, motion);
		return rtm::qvv_mul(relative(resumed, to), motion);
	}

	struct extract_args
	{
		const compressed_tracks* tracks;
		uint32_t rounding;
		const uint8_t* per_track_rounding;
		const float* constant_defaults;
		const float* variable_defaults;
		uint32_t root;
		float times[4];			// from, to, the clamp duration, 0
		float* samples;			// [4][12]
	};

	template<class settings_type, class writer_type>
	int extract(const extract_args& args)
	{
		decompression_context<settings_type> context;
		if (!context.initialize(*args.tracks))
			return -1;
		context.set_looping_policy(sample_looping_policy::clamp);
		for (int i = 0; i < 4; ++i)
		{
			writer_type writer;
			writer.root = args.root;
			writer.row = args.samples + i * 12;
			writer.per_track_rounding = args.per_track_rounding;
			writer.variable_defaults = args.variable_defaults;
			if (args.constant_defaults != nullptr)
				std::memcpy(writer.constant_defaults, args.constant_defaults, sizeof(writer.constant_defaults));
			context.seek(args.times[i], static_cast<sample_rounding_policy>(args.rounding));
			context.decompress_tracks(writer);
		}
		return 0;
	}

	template<class settings_type>
	int extract_writer(uint32_t writer_mode, const extract_args& args)
	{
		switch (writer_mode)
		{
		case 0: return extract<settings_type, root_writer_legacy>(args);
		case 2: return extract<settings_type, root_writer_constant>(args);
		case 3: return extract<settings_type, root_writer_variable>(args);
		default: return -2;
		}
	}
}

extern "C"
{
	__attribute__((visibility("default"))) void aclref_qvv_inverse(const float* in, float* out)
	{
		store_row(rtm::qvv_inverse(load_row(in)), out);
	}

	__attribute__((visibility("default"))) void aclref_qvv_mul(const float* lhs, const float* rhs, float* out)
	{
		store_row(rtm::qvv_mul(load_row(lhs), load_row(rhs)), out);
	}

	// M from the four root samples T(from), T(to), T(D), T(0)
	__attribute__((visibility("default"))) void aclref_root_motion_compose(const float* from, const float* to, const float* end, const float* start,
		int32_t cycles, float* out)
	{
		store_row(compose(load_row(from), load_row(to), load_row(end), load_row(start), cycles), out);
	}

	// The whole path of one request: settings_kind as ref_tool.cpp (0 default, 1 debug, 2 benchmark, 3 never, 4 all lerp, 5 raw only),
	// writer_mode 0 legacy / 2 constant / 3 variable defaults. out_samples [4][12]: T(from), T(to), T(D), T(0); out [12]: M. Returns < 0 when
	// the clip does not initialise, the root is not one of its tracks or a mode is unknown.
	__attribute__((visibility("default"))) int aclref_extract_root_motion(const void* blob, uint32_t settings_kind, uint32_t writer_mode,
		uint32_t rounding, const uint8_t* per_track_rounding, const float* constant_defaults, const float* variable_defaults, uint32_t root,
		float from_time, float to_time, int32_t cycles, float* out_samples, float* out)
	{
		const compressed_tracks& tracks = *static_cast<const compressed_tracks*>(blob);
		if (root >= tracks.get_num_tracks())
			return -4;
		extract_args args;
		args.tracks = &tracks;
		args.rounding = rounding;
		args.per_track_rounding = per_track_rounding;
		args.constant_defaults = constant_defaults;
		args.variable_defaults = variable_defaults;
		args.root = root;
		args.times[0] = from_time;
		args.times[1] = to_time;
		args.times[2] = tracks.get_finite_duration(sample_looping_policy::clamp);
		args.times[3] = 0.0F;
		args.samples = out_samples;
		std::memset(out_samples, 0, 4 * 12 * sizeof(float));
		int status;
		switch (settings_kind)
		{
		case 0: status = extract_writer<default_transform_decompression_settings>(writer_mode, args); break;
		case 1: status = extract_writer<debug_transform_decompression_settings>(writer_mode, args); break;
		case 2: status = extract_writer<settings_benchmark>(writer_mode, args); break;
		case 3: status = extract_writer<settings_never>(writer_mode, args); break;
		case 4: status = extract_writer<settings_all_lerp>(writer_mode, args); break;
		case 5: status = extract_writer<settings_raw_only>(writer_mode, args); break;
		default: status = -3; break;
		}
		if (status != 0)
			return status;
		aclref_root_motion_compose(out_samples, out_samples + 12, out_samples + 24, out_samples + 36, cycles, out);
		return 0;
	}
}
