// oracle/ref_additive.cpp -- TEST INFRASTRUCTURE ONLY: additive clips and acl::apply_additive_to_base from the unmodified reference, compiled
// into _ref/libaclref_additive.so (oracle/additive.mk) where the reference tree exists. It compiles ref_tool.cpp in for the raw clip synthesis
// of a spec (make_transform_tracks) and its compression settings.
#include "ref_tool.cpp"

#include <acl/core/additive_utils.h>

extern "C"
{
	// An additive clip as the reference's compressor writes it: the raw clips of `base_spec` (the base) and `spec` (the full animation, same
	// track count) are synthesised, the additive raw track of each bone is convert_to_relative / convert_to_additive0 / convert_to_additive1
	// (additive_utils.h:176-194) of (base(sample), full(sample)) at every sample of the full clip (the base's last sample past its end), and
	// compress_track_list(allocator, additive, settings of `spec`, base, additive_format, ...) (compression/compress.h:82) compresses it.
	// Returns 0 on success; the blob is released with aclref_free().
	__attribute__((visibility("default"))) int aclref_compress_additive(const aclref_transform_spec* base_spec, const aclref_transform_spec* spec,
		uint32_t additive_format, void** out_blob, uint32_t* out_size)
	{
		if (base_spec->num_tracks != spec->num_tracks || additive_format < 1 || additive_format > 3)
			return -3;
		iallocator& alloc = allocator();
		track_array_qvvf base_list(alloc, base_spec->num_tracks);
		make_transform_tracks(*base_spec, base_list);
		track_array_qvvf full_list(alloc, spec->num_tracks);
		make_transform_tracks(*spec, full_list);

		const additive_clip_format8 format = static_cast<additive_clip_format8>(additive_format);
		track_array_qvvf additive_list(alloc, spec->num_tracks);
		for (uint32_t bone = 0; bone < spec->num_tracks; ++bone)
		{
			const track_qvvf& base = base_list[bone];
			const track_qvvf& full = full_list[bone];
			track_qvvf additive = track_qvvf::make_reserve(full.get_description(), alloc, spec->num_samples, spec->sample_rate);
			for (uint32_t sample = 0; sample < spec->num_samples; ++sample)
			{
				const rtm::qvvf base_sample = base[sample < base_spec->num_samples ? sample : base_spec->num_samples - 1];
				if (format == additive_clip_format8::relative)
					additive[sample] = convert_to_relative(base_sample, full[sample]);
				else if (format == additive_clip_format8::additive0)
					additive[sample] = convert_to_additive0(base_sample, full[sample]);
				else
					additive[sample] = convert_to_additive1(base_sample, full[sample]);
			}
			additive_list[bone] = std::move(additive);
		}

		qvvf_transform_error_metric error_metric;
		compression_settings settings;
		settings.level = static_cast<compression_level8>(spec->level);
		settings.rotation_format = static_cast<rotation_format8>(spec->rotation_format);
		settings.translation_format = static_cast<vector_format8>(spec->translation_format);
		settings.scale_format = static_cast<vector_format8>(spec->scale_format);
		settings.error_metric = &error_metric;
		settings.optimize_loops = spec->optimize_loops != 0;
		settings.keyframe_stripping.strip_trivial = spec->strip_trivial != 0;
		settings.keyframe_stripping.proportion = spec->strip_proportion;
		settings.keyframe_stripping.threshold = spec->strip_threshold;

		compressed_tracks* tracks = nullptr;
		output_stats stats;
		const error_result result = compress_track_list(alloc, additive_list, settings, base_list, format, tracks, stats);
		if (result.any() || tracks == nullptr)
		{
			fprintf(stderr, "aclref_compress_additive: %s\n", result.any() ? result.c_str() : "no output");
			return -1;
		}
		const uint32_t size = tracks->get_size();
		void* copy = nullptr;
		if (posix_memalign(&copy, 64, size + 64) != 0)
			return -2;
		std::memcpy(copy, tracks, size);
		std::memset(static_cast<uint8_t*>(copy) + size, 0, 64);
		alloc.deallocate(tracks, size);
		*out_blob = copy;
		*out_size = size;
		return 0;
	}

	// acl::apply_additive_to_base(format, base, additive) (additive_utils.h:152-162) on every bone of one pose: [num_tracks][12] rtm::qvvf
	// rows in, out [num_tracks][12] (rotation xyzw, translation xyz + w, scale xyz + w as rtm leaves them)
	__attribute__((visibility("default"))) void aclref_apply_additive_to_base(uint32_t additive_format, const float* base_pose, const float* additive_pose,
		uint32_t num_tracks, float* out)
	{
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			const float* b = base_pose + size_t(bone) * 12;
			const float* a = additive_pose + size_t(bone) * 12;
			const rtm::qvvf base = rtm::qvv_set(rtm::quat_load(b), rtm::vector_load(b + 4), rtm::vector_load(b + 8));
			const rtm::qvvf additive = rtm::qvv_set(rtm::quat_load(a), rtm::vector_load(a + 4), rtm::vector_load(a + 8));
			const rtm::qvvf result = apply_additive_to_base(static_cast<additive_clip_format8>(additive_format), base, additive);
			float* o = out + size_t(bone) * 12;
			rtm::quat_store(result.rotation, o);
			rtm::vector_store(result.translation, o + 4);
			rtm::vector_store(result.scale, o + 8);
		}
	}
}
