// tests/cpp/shim_skinning.cpp -- acl_b200::batch_decompressor's four skinning members against the C calls they wrap: the clip decoded
// plain, as additive pairs (additive0, the clip over itself) and as blend pairs, with a binary tree skeleton and random inverse binds, then
// the standalone call on the local rows, in place through the shim; the outputs must be byte-identical.
// usage: shim_skinning <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
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
		const uint32_t num_requests = 64;
		std::vector<aclb200_request> requests;
		std::vector<aclb200_blend_request> pairs;
		for (uint32_t i = 0; i < num_requests; ++i)
		{
			requests.push_back(aclb200_request{ 0u, float(i) * 0.037f - 0.1f });
			pairs.push_back(aclb200_blend_request{ aclb200_request{ 0u, float(i) * 0.037f - 0.1f }, aclb200_request{ 0u, float(63 - i) * 0.029f } });
		}
		std::vector<uint32_t> parents(num_tracks);
		std::vector<float> inverse_bind(size_t(num_tracks) * 12);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
			// a scaled shear plus a translation: x_axis, y_axis, z_axis, w_axis
			const float s = 0.5f + 0.01f * float(bone);
			const float axes[12] = { s, 0.1f, 0.0f, 0.0f, s, -0.2f, 0.05f, 0.0f, -s, float(bone) * 0.1f, -1.0f, 0.25f };
			std::memcpy(&inverse_bind[size_t(bone) * 12], axes, sizeof(axes));
		}
		const size_t out_bytes = size_t(num_tracks) * 48 * num_requests;
		aclb200_request* d_requests = nullptr;
		aclb200_blend_request* d_pairs = nullptr;
		uint32_t* d_parents = nullptr;
		float* d_inverse_bind = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, num_requests * sizeof(aclb200_request)) != cudaSuccess || cudaMalloc(&d_pairs, num_requests * sizeof(aclb200_blend_request)) != cudaSuccess
			|| cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&d_inverse_bind, inverse_bind.size() * sizeof(float)) != cudaSuccess
			|| cudaMalloc(&d_out[0], out_bytes) != cudaSuccess || cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), num_requests * sizeof(aclb200_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_pairs, pairs.data(), num_requests * sizeof(aclb200_blend_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_inverse_bind, inverse_bind.data(), inverse_bind.size() * sizeof(float), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
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
		const auto reset = [&]()
		{
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xCD, out_bytes);
		};

		reset();
		batch.decompress_tracks_skinning(d_requests, num_requests, options, d_parents, nullptr, d_inverse_bind, d_out[0]);
		if (aclb200_decompress_tracks_skinning(device.get(), batch.clipset(), d_requests, num_requests, &options, d_parents, nullptr, d_inverse_bind,
			d_out[1], nullptr, nullptr) != ACLB200_OK || !same("decompress_tracks_skinning"))
			return 1;

		// an aclb200_blend_request and an aclb200_additive_request are the same two requests back to back
		const aclb200_additive_request* d_additive = reinterpret_cast<const aclb200_additive_request*>(d_pairs);
		reset();
		batch.decompress_tracks_additive_skinning(d_additive, num_requests, options, ACLB200_ADDITIVE_ADDITIVE0, nullptr, d_parents, nullptr, d_inverse_bind,
			d_out[0]);
		if (aclb200_decompress_tracks_additive_skinning(device.get(), batch.clipset(), d_additive, num_requests, &options, ACLB200_ADDITIVE_ADDITIVE0, nullptr,
			d_parents, nullptr, d_inverse_bind, d_out[1], nullptr, nullptr) != ACLB200_OK || !same("decompress_tracks_additive_skinning"))
			return 1;

		reset();
		batch.decompress_tracks_blend_skinning(d_pairs, num_requests, options, 0.3f, nullptr, d_parents, nullptr, d_inverse_bind, d_out[0]);
		if (aclb200_decompress_tracks_blend_skinning(device.get(), batch.clipset(), d_pairs, num_requests, &options, 0.3f, nullptr, d_parents, nullptr,
			d_inverse_bind, d_out[1], nullptr, nullptr) != ACLB200_OK || !same("decompress_tracks_blend_skinning"))
			return 1;

		// the standalone call over the local rows: in place through the shim, into the other buffer through the C call; both equal the
		// fused call
		batch.decompress_tracks(d_requests, num_requests, options, d_out[0]);
		cudaMemcpy(d_out[1], d_out[0], out_bytes, cudaMemcpyDeviceToDevice);
		batch.local_to_skinning(d_out[0], d_out[0], num_requests, num_tracks, d_parents, d_inverse_bind);
		uint8_t* d_local = d_out[1];
		if (cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		if (aclb200_local_to_skinning(device.get(), d_local, d_out[1], num_requests, num_tracks, 0, d_parents, d_inverse_bind, nullptr, nullptr) != ACLB200_OK
			|| !same("local_to_skinning"))
			return 1;
		batch.decompress_tracks_skinning(d_requests, num_requests, options, d_parents, nullptr, d_inverse_bind, d_out[1]);
		if (!same("local_to_skinning against decompress_tracks_skinning"))
			return 1;
		cudaFree(d_local);
		cudaFree(d_requests);
		cudaFree(d_pairs);
		cudaFree(d_parents);
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
