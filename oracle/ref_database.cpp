// oracle/ref_database.cpp -- TEST INFRASTRUCTURE ONLY: the reference's streaming database path, compiled with every entry point of
// ref_tool.cpp into _ref/libaclref_db.so (oracle/database.mk).
//
//   aclref_build_database            compress N clips with database support and split them with acl::build_database
//                                    (compression/compress.h:86-100) into the bound clips and one compressed_database
//   aclref_decompress_tracks_database decompression_context<settings_database>::initialize(tracks, db) (decompress.impl.h:85-110) where
//                                    db is a database_context driven by memcpy streamers (debug_database_streamer) through a sequence of
//                                    stream_in / stream_out(tier, n) calls; then seek + decompress_tracks / decompress_track
#include "ref_tool.cpp"

#include <acl/decompression/database/impl/debug_database_streamer.h>

namespace
{
	void* copy_out(const void* src, uint32_t size)
	{
		void* copy = nullptr;
		if (posix_memalign(&copy, 64, size + 64) != 0)
			return nullptr;
		std::memcpy(copy, src, size);
		std::memset(static_cast<uint8_t*>(copy) + size, 0, 64);
		return copy;
	}
}

extern "C"
{
	// out_clips[i] / out_clip_sizes[i]: clip i bound to the database; *out_database: the database (inline bulk data). Free with aclref_free.
	int aclref_build_database(const aclref_transform_spec* specs, uint32_t num_clips, float medium_proportion, float low_proportion,
		uint32_t max_chunk_size, void** out_clips, uint32_t* out_clip_sizes, void** out_database, uint32_t* out_database_size)
	{
		iallocator& alloc = allocator();
		std::vector<compressed_tracks*> inputs(num_clips, nullptr);
		for (uint32_t clip = 0; clip < num_clips; ++clip)
		{
			track_array_qvvf track_list(alloc, specs[clip].num_tracks);
			make_transform_tracks(specs[clip], track_list);
			qvvf_transform_error_metric error_metric;
			compression_settings settings;
			settings.level = static_cast<compression_level8>(specs[clip].level);
			settings.rotation_format = static_cast<rotation_format8>(specs[clip].rotation_format);
			settings.translation_format = static_cast<vector_format8>(specs[clip].translation_format);
			settings.scale_format = static_cast<vector_format8>(specs[clip].scale_format);
			settings.error_metric = &error_metric;
			settings.optimize_loops = specs[clip].optimize_loops != 0;
			settings.enable_database_support = true;
			output_stats stats;
			const error_result result = compress_track_list(alloc, track_list, settings, inputs[clip], stats);
			if (result.any() || inputs[clip] == nullptr)
			{
				fprintf(stderr, "aclref_build_database: clip %u: %s\n", clip, result.any() ? result.c_str() : "no output");
				return -1;
			}
		}

		compression_database_settings database_settings;
		database_settings.medium_importance_tier_proportion = medium_proportion;
		database_settings.low_importance_tier_proportion = low_proportion;
		if (max_chunk_size != 0)
			database_settings.max_chunk_size = max_chunk_size;
		std::vector<compressed_tracks*> bound(num_clips, nullptr);
		compressed_database* database = nullptr;
		const error_result result = build_database(alloc, database_settings, const_cast<const compressed_tracks**>(inputs.data()), num_clips, bound.data(), database);
		for (compressed_tracks* tracks : inputs)
			alloc.deallocate(tracks, tracks->get_size());
		if (result.any() || database == nullptr)
		{
			fprintf(stderr, "aclref_build_database: %s\n", result.any() ? result.c_str() : "no output");
			return -2;
		}
		for (uint32_t clip = 0; clip < num_clips; ++clip)
		{
			out_clip_sizes[clip] = bound[clip]->get_size();
			out_clips[clip] = copy_out(bound[clip], out_clip_sizes[clip]);
			alloc.deallocate(bound[clip], bound[clip]->get_size());
		}
		*out_database_size = database->get_size();
		*out_database = copy_out(database, *out_database_size);
		alloc.deallocate(database, database->get_size());
		return 0;
	}

	// ops: num_ops triples (0 = stream_in / 1 = stream_out, tier 1 medium / 2 low, num_chunks). track_index < 0: decompress_tracks.
	int aclref_decompress_tracks_database(const void* clip_blob, const void* database_blob, const uint32_t* ops, uint32_t num_ops,
		float sample_time, uint32_t rounding, uint32_t looping, int32_t track_index, float* out)
	{
		iallocator& alloc = allocator();
		const compressed_tracks& tracks = *static_cast<const compressed_tracks*>(clip_blob);
		const compressed_database& database = *static_cast<const compressed_database*>(database_blob);
		debug_database_streamer medium(alloc, database.get_bulk_data(quality_tier::medium_importance), database.get_bulk_data_size(quality_tier::medium_importance));
		debug_database_streamer low(alloc, database.get_bulk_data(quality_tier::lowest_importance), database.get_bulk_data_size(quality_tier::lowest_importance));
		database_context<default_database_settings> db;
		if (!db.initialize(alloc, database, medium, low))
			return -1;
		for (uint32_t op = 0; op < num_ops; ++op)
		{
			const quality_tier tier = static_cast<quality_tier>(ops[3 * op + 1]);
			if (ops[3 * op] == 0)
				db.stream_in(tier, ops[3 * op + 2]);
			else
				db.stream_out(tier, ops[3 * op + 2]);
		}
		decompression_context<settings_database> context;
		if (!context.initialize(tracks, db))
			return -2;
		context.set_looping_policy(static_cast<sample_looping_policy>(looping));
		pose_writer_legacy writer;
		writer.out = out;
		context.seek(sample_time, static_cast<sample_rounding_policy>(rounding));
		if (track_index < 0)
			context.decompress_tracks(writer);
		else
			context.decompress_track(uint32_t(track_index), writer);
		return 0;
	}
}
