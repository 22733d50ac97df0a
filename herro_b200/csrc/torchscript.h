// TorchScript archive reader (torchscript.cpp): parameters of a `torch.jit.save`d module, by state_dict name.
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

namespace hb {

struct TsTensor { std::vector<int64_t> shape; std::vector<float> data; };  // contiguous, converted to fp32
struct TsModel {
    std::map<std::string, TsTensor> tensors;   // "layers.0.qkv.weight" -> ...
    std::map<std::string, int64_t> ints;       // integer attributes of the module tree ("layers.0.H")
    std::string err;
};
struct TsDims { int stem_k = 0, channels = 0, heads = 0, layers = 0, ffn = 0, collapse = 0, pos_layers = 0, pos_heads = 0, pos_ffn = 0; };

bool ts_is_zip(const uint8_t* buf, size_t n);
bool ts_read_archive(const uint8_t* buf, size_t n, TsModel& out);
// oracle/forward_ref.HerroNet naming -> the tensor names / forms of the HB200W1 blob (herro_b200/weights.py)
bool ts_to_canonical(const TsModel& m, int heads_hint, TsDims& d, std::map<std::string, std::vector<float>>& T, std::string& err);

}  // namespace hb
