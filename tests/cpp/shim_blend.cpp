// tests/cpp/shim_blend.cpp -- acl_b200::batch_decompressor::decompress_tracks_blend and blend_poses against the C calls they wrap: the clip
// blended with itself at other sample times, with a weight per pair and with the scalar weight, local rows and object space rows (a binary
// tree), then the standalone call on the local rows; the outputs must be byte-identical.
// usage: shim_blend <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
#include "../../include/acl_b200/decompress.h"

#include <cuda_runtime.h>

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
		std::vector<aclb200_blend_request> requests;
		std::vector<float> weights;
		for (uint32_t i = 0; i < 64; ++i)
		{
			requests.push_back(aclb200_blend_request{ aclb200_request{ 0u, float(i) * 0.037f - 0.1f }, aclb200_request{ 0u, float(63 - i) * 0.029f } });
			weights.push_back(float(i) / 42.0f - 0.25f);
		}
		std::vector<uint32_t> parents(num_tracks);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
		const size_t out_bytes = size_t(num_tracks) * 48 * requests.size();
		aclb200_blend_request* d_requests = nullptr;
		uint32_t* d_parents = nullptr;
		float* d_weights = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_blend_request)) != cudaSuccess || cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_weights, weights.size() * sizeof(float)) != cudaSuccess || cudaMalloc(&d_out[0], out_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_blend_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_weights, weights.data(), weights.size() * sizeof(float), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		const uint32_t num_requests = uint32_t(requests.size());
		const auto same = [&](const char* what) -> bool
		{
			std::vector<uint8_t> got[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(got[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return false;
			if (std::memcmp(got[0].data(), got[1].data(), out_bytes) == 0)
				return true;
			std::printf("FAIL %s\n", what);
			return false;
		};
		for (const float* weight_pointer : { static_cast<const float*>(nullptr), static_cast<const float*>(d_weights) })
		{
			for (const uint32_t* parent_pointer : { static_cast<const uint32_t*>(nullptr), static_cast<const uint32_t*>(d_parents) })
			{
				cudaMemset(d_out[0], 0xAB, out_bytes);
				cudaMemset(d_out[1], 0xCD, out_bytes);
				batch.decompress_tracks_blend(d_requests, num_requests, options, 0.3f, weight_pointer, d_out[0], parent_pointer);
				if (aclb200_decompress_tracks_blend(device.get(), batch.clipset(), d_requests, num_requests, &options, 0.3f, weight_pointer, parent_pointer,
					nullptr, ACLB200_OBJECT_QVVF, d_out[1], nullptr, nullptr) != ACLB200_OK)
					return 1;
				if (!same(parent_pointer != nullptr ? "object space" : "local"))
					return 1;
			}
			// the standalone call over the local rows: in place through the shim, into the other buffer through the C call
			batch.decompress_tracks_blend(d_requests, num_requests, options, 0.3f, weight_pointer, d_out[0]);
			cudaMemcpy(d_out[1], d_out[0], out_bytes, cudaMemcpyDeviceToDevice);
			batch.blend_poses(d_out[0], d_out[0] + out_bytes / 2, d_out[0], num_requests / 2, num_tracks, 0.7f, weight_pointer);
			if (aclb200_blend_poses(device.get(), d_out[1], d_out[1] + out_bytes / 2, d_out[1], num_requests / 2, num_tracks, 0, 0.7f, weight_pointer,
				nullptr) != ACLB200_OK)
				return 1;
			if (!same("blend_poses"))
				return 1;
		}
		cudaFree(d_requests);
		cudaFree(d_parents);
		cudaFree(d_weights);
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
