// tests/cpp/shim_masked_layers.cpp -- acl_b200::batch_decompressor::decompress_tracks_layered_masked and
// decompress_tracks_layered_masked_skinning against the C calls they wrap: the clip stacked on itself four layers deep (base, BLEND under
// an upper/lower mask, OFF, ADDITIVE relative at weight 0.5 under a feathered mask) at other sample times, local rows, object space rows
// and skinning rows (a binary tree, identity inverse binds); the outputs must be byte-identical.
// usage: shim_masked_layers <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
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
		const uint32_t num_layers = 4;
		std::vector<aclb200_layer> layers;
		std::vector<uint32_t> layer_masks;
		for (uint32_t i = 0; i < 64; ++i)
		{
			layers.push_back(aclb200_layer{ aclb200_request{ 0u, float(i) * 0.037f - 0.1f }, ACLB200_LAYER_BLEND, 0.0f });
			layers.push_back(aclb200_layer{ aclb200_request{ 0u, float(63 - i) * 0.029f }, ACLB200_LAYER_BLEND, float(i) / 63.0f });
			layers.push_back(aclb200_layer{ aclb200_request{ 0xFFFFFFFFu, 0.0f }, ACLB200_LAYER_OFF, 0.0f });
			layers.push_back(aclb200_layer{ aclb200_request{ 0u, float(i) * 0.011f }, ACLB200_LAYER_ADDITIVE, 0.5f });
			layer_masks.insert(layer_masks.end(), { ACLB200_LAYER_NO_MASK, 0u, ACLB200_LAYER_NO_MASK, (i & 1) != 0 ? 1u : ACLB200_LAYER_NO_MASK });
		}
		// mask 0: the upper half of the bones 1, the rest 0; mask 1: a ramp from 0 to 1
		std::vector<float> bone_masks(size_t(num_tracks) * 2);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			bone_masks[bone] = bone >= num_tracks / 2 ? 1.0f : 0.0f;
			bone_masks[num_tracks + bone] = float(bone) / float(num_tracks);
		}
		const uint32_t num_poses = uint32_t(layers.size()) / num_layers;
		std::vector<uint32_t> parents(num_tracks);
		std::vector<float> inverse_bind(size_t(num_tracks) * 12, 0.0f);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
			inverse_bind[bone * 12 + 0] = inverse_bind[bone * 12 + 4] = inverse_bind[bone * 12 + 8] = 1.0f;
		}
		const size_t out_bytes = size_t(num_tracks) * 48 * num_poses;
		aclb200_layer* d_layers = nullptr;
		uint32_t* d_layer_masks = nullptr;
		float* d_bone_masks = nullptr;
		uint32_t* d_parents = nullptr;
		float* d_inverse_bind = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_layers, layers.size() * sizeof(aclb200_layer)) != cudaSuccess || cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_layer_masks, layer_masks.size() * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_bone_masks, bone_masks.size() * sizeof(float)) != cudaSuccess
			|| cudaMalloc(&d_inverse_bind, inverse_bind.size() * sizeof(float)) != cudaSuccess || cudaMalloc(&d_out[0], out_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_layers, layers.data(), layers.size() * sizeof(aclb200_layer), cudaMemcpyHostToDevice);
		cudaMemcpy(d_layer_masks, layer_masks.data(), layer_masks.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_bone_masks, bone_masks.data(), bone_masks.size() * sizeof(float), cudaMemcpyHostToDevice);
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
		for (const uint32_t* parent_pointer : { static_cast<const uint32_t*>(nullptr), static_cast<const uint32_t*>(d_parents) })
		{
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xCD, out_bytes);
			batch.decompress_tracks_layered_masked(d_layers, d_layer_masks, num_poses, num_layers, d_bone_masks, 2, 0, options,
				ACLB200_ADDITIVE_RELATIVE, nullptr, d_out[0], parent_pointer);
			if (aclb200_decompress_tracks_layered_masked(device.get(), batch.clipset(), d_layers, d_layer_masks, num_poses, num_layers, d_bone_masks,
				2, 0, &options, ACLB200_ADDITIVE_RELATIVE, nullptr, parent_pointer, nullptr, ACLB200_OBJECT_QVVF, d_out[1], nullptr, nullptr) != ACLB200_OK)
				return 1;
			if (!same(parent_pointer != nullptr ? "object space" : "local"))
				return 1;
		}
		cudaMemset(d_out[0], 0xAB, out_bytes);
		cudaMemset(d_out[1], 0xCD, out_bytes);
		batch.decompress_tracks_layered_masked_skinning(d_layers, d_layer_masks, num_poses, num_layers, d_bone_masks, 2, num_tracks, options,
			ACLB200_ADDITIVE_RELATIVE, nullptr, d_parents, nullptr, d_inverse_bind, d_out[0]);
		if (aclb200_decompress_tracks_layered_masked_skinning(device.get(), batch.clipset(), d_layers, d_layer_masks, num_poses, num_layers,
			d_bone_masks, 2, num_tracks, &options, ACLB200_ADDITIVE_RELATIVE, nullptr, d_parents, nullptr, d_inverse_bind, d_out[1], nullptr,
			nullptr) != ACLB200_OK)
			return 1;
		if (!same("skinning"))
			return 1;
		cudaFree(d_layers);
		cudaFree(d_layer_masks);
		cudaFree(d_bone_masks);
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
