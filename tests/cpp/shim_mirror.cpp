// tests/cpp/shim_mirror.cpp -- acl_b200::batch_decompressor::mirror_poses, decompress_tracks_mirrored and decompress_tracks_mirrored_skinning
// against the C calls they wrap: a clip decoded at 64 times with every other request mirrored (a table pairing bones (0,1), (2,3) .. with
// fabricated corrections), as local rows, object space rows and skinning rows (a binary tree, identity inverse binds), and the local rows
// mirrored again on the device with a per-pose flag; the outputs must be byte-identical.
// usage: shim_mirror <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
#include "../../include/acl_b200/decompress.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

int main(int argc, char** argv)
{
	if (argc != 2)
		return 2;
	std::ifstream file(argv[1], std::ios::binary);
	const std::vector<char> blob((std::istreambuf_iterator<char>(file)), std::istreambuf_iterator<char>());
	try
	{
		acl_b200::device_context device(0);
		acl_b200::batch_decompressor batch(device);
		const void* pointer = blob.data();
		const uint32_t size = uint32_t(blob.size());
		if (!batch.upload(&pointer, &size, 1))
			return 1;
		const uint32_t num_tracks = batch.info().max_tracks;
		const uint32_t num_poses = 64;
		std::vector<aclb200_mirrored_request> requests;
		std::vector<uint32_t> flags(num_poses);
		for (uint32_t i = 0; i < num_poses; ++i)
		{
			requests.push_back(aclb200_mirrored_request{ aclb200_request{ 0u, float(i) * 0.031f }, i % 2 });
			flags[i] = i % 3 == 2 ? 7u : i % 3;
		}
		std::vector<aclb200_mirror_entry> table(num_tracks);
		std::vector<uint32_t> parents(num_tracks);
		std::vector<float> inverse_bind(size_t(num_tracks) * 12, 0.0f);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			aclb200_mirror_entry& e = table[bone];
			const float a = std::sin(float(bone) * 0.7f), b = std::cos(float(bone) * 0.7f);
			const float pre[4] = { a * 0.6f, 0.0f, a * 0.8f, b };
			const float post[4] = { 0.0f, b, 0.0f, a };
			std::memcpy(e.pre, pre, sizeof(pre));
			std::memcpy(e.post, post, sizeof(post));
			e.mirror = (bone ^ 1u) < num_tracks ? bone ^ 1u : bone;
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
			inverse_bind[bone * 12 + 0] = inverse_bind[bone * 12 + 4] = inverse_bind[bone * 12 + 8] = 1.0f;
		}
		const size_t out_bytes = size_t(num_tracks) * 48 * num_poses;
		aclb200_mirrored_request* d_requests = nullptr;
		aclb200_mirror_entry* d_table = nullptr;
		uint32_t* d_parents = nullptr;
		uint32_t* d_flags = nullptr;
		float* d_inverse_bind = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_mirrored_request)) != cudaSuccess
			|| cudaMalloc(&d_table, table.size() * sizeof(aclb200_mirror_entry)) != cudaSuccess
			|| cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&d_flags, num_poses * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_inverse_bind, inverse_bind.size() * sizeof(float)) != cudaSuccess || cudaMalloc(&d_out[0], out_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_mirrored_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_table, table.data(), table.size() * sizeof(aclb200_mirror_entry), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_flags, flags.data(), num_poses * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_inverse_bind, inverse_bind.data(), inverse_bind.size() * sizeof(float), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		std::vector<uint8_t> out[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
		auto same = [&]() {
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(out[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return false;
			return std::memcmp(out[0].data(), out[1].data(), out_bytes) == 0;
		};
		for (int route = 0; route < 4; ++route)
		{
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xAB, out_bytes);
			aclb200_status status = ACLB200_OK;
			if (route == 0)
			{
				batch.decompress_tracks_mirrored(d_requests, num_poses, options, d_table, ACLB200_MIRROR_X, d_out[0]);
				status = aclb200_decompress_tracks_mirrored(device.get(), batch.clipset(), d_requests, num_poses, &options, d_table, ACLB200_MIRROR_X,
					nullptr, nullptr, ACLB200_OBJECT_QVVF, d_out[1], nullptr, nullptr);
			}
			else if (route == 1)
			{
				batch.decompress_tracks_mirrored(d_requests, num_poses, options, d_table, ACLB200_MIRROR_Y, d_out[0], d_parents, nullptr,
					ACLB200_OBJECT_MATRIX3X4F);
				status = aclb200_decompress_tracks_mirrored(device.get(), batch.clipset(), d_requests, num_poses, &options, d_table, ACLB200_MIRROR_Y,
					d_parents, nullptr, ACLB200_OBJECT_MATRIX3X4F, d_out[1], nullptr, nullptr);
			}
			else if (route == 2)
			{
				batch.decompress_tracks_mirrored_skinning(d_requests, num_poses, options, d_table, ACLB200_MIRROR_Z, d_parents, d_inverse_bind, d_out[0]);
				status = aclb200_decompress_tracks_mirrored_skinning(device.get(), batch.clipset(), d_requests, num_poses, &options, d_table,
					ACLB200_MIRROR_Z, d_parents, nullptr, d_inverse_bind, d_out[1], nullptr, nullptr);
			}
			else
			{
				// local rows decoded into both outputs, then mirrored in place with the per-pose flags
				batch.decompress_tracks_mirrored(d_requests, num_poses, options, d_table, ACLB200_MIRROR_X, d_out[0]);
				batch.decompress_tracks_mirrored(d_requests, num_poses, options, d_table, ACLB200_MIRROR_X, d_out[1]);
				batch.mirror_poses(d_out[0], d_out[0], num_poses, num_tracks, d_table, ACLB200_MIRROR_X, d_flags);
				status = aclb200_mirror_poses(device.get(), d_out[1], d_out[1], num_poses, num_tracks, 0, d_flags, d_table, ACLB200_MIRROR_X, nullptr,
					nullptr);
			}
			if (status != ACLB200_OK)
				return 1;
			if (!same())
			{
				std::printf("FAIL shim and C call differ (route %d)\n", route);
				return 1;
			}
		}
		cudaFree(d_requests);
		cudaFree(d_table);
		cudaFree(d_parents);
		cudaFree(d_flags);
		cudaFree(d_inverse_bind);
		cudaFree(d_out[0]);
		cudaFree(d_out[1]);
	}
	catch (const acl_b200::error& e)
	{
		std::fprintf(stderr, "%s\n", e.what());
		return e.status == ACLB200_ERR_NO_DEVICE ? 3 : 1;
	}
	std::printf("PASS\n");
	return 0;
}
