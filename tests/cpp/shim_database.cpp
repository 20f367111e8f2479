// tests/cpp/shim_database.cpp -- a REFERENCE call site of the streaming database API compiled against both namespaces.
//
// `decode()` is written once: database_context<settings>::initialize / stream_in / stream_out, decompression_context::initialize(tracks,
// database), seek, decompress_tracks into acl::acl_impl::debug_track_writer. It is instantiated with the acl:: classes and with the
// acl_b200:: classes. The reference's streamer-less database_context streams every chunk in (database.impl.h:91-212); its streaming
// flavour is driven by memcpy streamers (debug_database_streamer) over the database's inline bulk data.
//
// usage: shim_database <clip.acl.bin> <database.bin>
//   exit 0 = every pose bit-identical in every tier state, 3 = no usable GPU (no CPU fallback), 1 = mismatch.
#include <acl/core/ansi_allocator.h>
#include <acl/core/impl/debug_track_writer.h>
#include <acl/decompression/database/database.h>
#include <acl/decompression/database/impl/debug_database_streamer.h>
#include <acl/decompression/decompress.h>

#include "../../include/acl_b200/decompress.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

#if !ACLB200_WITH_ACL_HEADERS
	#error "this test must be compiled with the reference's headers on the include path"
#endif

namespace
{
	struct settings_database final : public acl::debug_transform_decompression_settings
	{
		using database_settings_type = acl::default_database_settings;
	};

	std::vector<uint8_t> read_file(const char* path)
	{
		std::ifstream file(path, std::ios::binary);
		std::vector<char> bytes((std::istreambuf_iterator<char>(file)), std::istreambuf_iterator<char>());
		std::vector<uint8_t> out(bytes.size() + 80, 0);
		std::memcpy(out.data(), bytes.data(), bytes.size());
		return out;
	}

	void report(const std::vector<float>& want, const std::vector<float>& got, const char* state, int& failures)
	{
		++failures;
		size_t index = 0;
		while (index < want.size() && index < got.size() && want[index] == got[index])
			++index;
		std::printf("%s: %zu / %zu values, first difference at %zu: %.9g vs %.9g\n", state, want.size(), got.size(), index,
			index < want.size() ? want[index] : 0.0, index < got.size() ? got[index] : 0.0);
	}

	template<class context_type, class database_type>
	std::vector<float> decode(acl::iallocator& allocator, const acl::compressed_tracks& tracks, const database_type& database, const float* times, int num_times)
	{
		context_type context;
		std::vector<float> poses;
		if (!context.initialize(tracks, database))
			return poses;
		acl::acl_impl::debug_track_writer writer(allocator, acl::track_type8::qvvf, tracks.get_num_tracks());
		for (int i = 0; i < num_times; ++i)
			for (int rounding = 0; rounding < 4; ++rounding)
			{
				// lanes a decode leaves unwritten (the scale of a clip without scale, with this writer) read as zero in both runs
				std::memset(writer.tracks_typed.qvvf, 0, sizeof(float) * 12 * tracks.get_num_tracks());
				context.seek(times[i], static_cast<acl::sample_rounding_policy>(rounding));
				context.decompress_tracks(writer);
				// rotation xyzw, translation xyz, scale xyz: the w lanes of translation and scale are not part of the decoded value
				const float* values = reinterpret_cast<const float*>(writer.tracks_typed.qvvf);
				for (uint32_t track = 0; track < tracks.get_num_tracks(); ++track)
					for (int lane : { 0, 1, 2, 3, 4, 5, 6, 8, 9, 10 })
						poses.push_back(values[track * 12 + lane]);
			}
		return poses;
	}
}

int main(int argc, char** argv)
{
	if (argc < 3)
		return 2;
	std::vector<uint8_t> clip_bytes = read_file(argv[1]);
	std::vector<uint8_t> database_bytes = read_file(argv[2]);
	// 16 byte aligned copies (compressed_tracks.h:53, compressed_database.h:52)
	std::vector<uint8_t> clip_store(clip_bytes.size() + 16), database_store(database_bytes.size() + 16);
	uint8_t* clip_aligned = clip_store.data() + ((16 - reinterpret_cast<uintptr_t>(clip_store.data()) % 16) % 16);
	uint8_t* database_aligned = database_store.data() + ((16 - reinterpret_cast<uintptr_t>(database_store.data()) % 16) % 16);
	std::memcpy(clip_aligned, clip_bytes.data(), clip_bytes.size());
	std::memcpy(database_aligned, database_bytes.data(), database_bytes.size());
	const acl::compressed_tracks& tracks = *reinterpret_cast<const acl::compressed_tracks*>(clip_aligned);
	const acl::compressed_database& database = *reinterpret_cast<const acl::compressed_database*>(database_aligned);
	const float times[] = { 0.0F, 0.13F, 0.5F, 0.77F, 1.01F, 2.2F };
	const int num_times = 6;
	acl::ansi_allocator allocator;
	int failures = 0;

	try
	{
		// 1. initialize(database) with inline bulk data: every chunk streamed in
		acl::database_context<acl::default_database_settings> reference_all;
		acl_b200::database_context<acl::default_database_settings> shim;
		if (!reference_all.initialize(allocator, database) || !shim.initialize(database))
			return 1;
		if (!shim.contains(tracks) || !shim.is_streamed_in(acl::quality_tier::medium_importance))
			++failures;
		const std::vector<float> want_all = decode<acl::decompression_context<settings_database>>(allocator, tracks, reference_all, times, num_times);
		const std::vector<float> got_all = decode<acl_b200::decompression_context<settings_database>>(allocator, tracks, shim, times, num_times);
		if (want_all.empty() || want_all != got_all)
			report(want_all, got_all, "every chunk streamed in", failures);

		// 2. the same calls on a streaming reference context and on the shim: everything out, then some medium, then all low
		acl::debug_database_streamer medium(allocator, database.get_bulk_data(acl::quality_tier::medium_importance), database.get_bulk_data_size(acl::quality_tier::medium_importance));
		acl::debug_database_streamer low(allocator, database.get_bulk_data(acl::quality_tier::lowest_importance), database.get_bulk_data_size(acl::quality_tier::lowest_importance));
		acl::database_context<acl::default_database_settings> reference;
		if (!reference.initialize(allocator, database, medium, low))
			return 1;
		shim.stream_out(acl::quality_tier::medium_importance);
		shim.stream_out(acl::quality_tier::lowest_importance);
		const struct { acl::quality_tier tier; uint32_t chunks; } steps[] = { { acl::quality_tier::medium_importance, 1 }, { acl::quality_tier::lowest_importance, ~0u } };
		for (const auto& step : steps)
		{
			const acl::database_stream_request_result want_result = reference.stream_in(step.tier, step.chunks);
			const acl::database_stream_request_result got_result = shim.stream_in(step.tier, step.chunks);
			if (want_result != got_result)
				++failures;
			const std::vector<float> want = decode<acl::decompression_context<settings_database>>(allocator, tracks, reference, times, num_times);
			const std::vector<float> got = decode<acl_b200::decompression_context<settings_database>>(allocator, tracks, shim, times, num_times);
			if (want.empty() || want != got)
				report(want, got, "streamed in step by step", failures);
		}
	}
	catch (const acl_b200::error& e)
	{
		std::printf("%s\n", e.what());
		return e.status == ACLB200_ERR_NO_DEVICE ? 3 : 1;
	}
	std::printf("%s: %d failure(s)\n", failures == 0 ? "PASS" : "FAIL", failures);
	return failures == 0 ? 0 : 1;
}
