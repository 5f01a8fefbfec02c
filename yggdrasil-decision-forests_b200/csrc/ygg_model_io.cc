// ygg_model_io.cc — writes a trained forest as a YDF model directory so that the reference's
// model::LoadModel reads it back (model/gradient_boosted_trees/gradient_boosted_trees.cc:111-139):
//     header.pb                           model::proto::AbstractModel        (model/abstract_model.proto)
//     data_spec.pb                        dataset::proto::DataSpecification  (dataset/data_spec.proto)
//     gradient_boosted_trees_header.pb    gradient_boosted_trees::proto::Header
//     nodes-00000-of-00001                blob sequence of decision_tree::proto::Node, pre-order
//                                         (utils/blob_sequence.h:121-149, decision_tree.cc:609-646)
//     done                                empty marker
// protoc is not available in this image: the handful of messages is emitted with a minimal proto2
// wire encoder (varint / fixed32 / fixed64 / length-delimited).  Field numbers are cited inline.
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "../../include/ygg_b200.h"
#include "../../include/ygg_b200_model.h"

namespace {

struct Pb {
  std::string s;
  void varint(uint64_t v) {
    while (v >= 0x80) { s.push_back(static_cast<char>(v | 0x80)); v >>= 7; }
    s.push_back(static_cast<char>(v));
  }
  void key(int field, int wire) { varint(static_cast<uint64_t>(field) << 3 | wire); }
  void i64(int field, int64_t v) { key(field, 0); varint(static_cast<uint64_t>(v)); }  // int32/int64/bool/enum
  void f32(int field, float v) { key(field, 5); s.append(reinterpret_cast<const char*>(&v), 4); }
  void f64(int field, double v) { key(field, 1); s.append(reinterpret_cast<const char*>(&v), 8); }
  void bytes(int field, const std::string& b) { key(field, 2); varint(b.size()); s.append(b); }
  void msg(int field, const Pb& m) { bytes(field, m.s); }
};

bool write_file(const std::string& path, const std::string& data) {
  FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  const bool ok = data.empty() || std::fwrite(data.data(), 1, data.size(), f) == data.size();
  return std::fclose(f) == 0 && ok;
}

// decision_tree::proto::Node for one flat node (model/decision_tree/decision_tree.proto).
// `set`: the positive set of a wide categorical split (null: n.cat_mask, 256 categories at most).
std::string encode_node(const ygg_node& n, int use_hessian_gain, const int32_t* feature_col_idx,
                        const int32_t* feature_num_values, const uint32_t* set) {
  Pb reg;  // NodeRegressorOutput
  reg.f32(1, n.leaf_value);  // top_value
  if (use_hessian_gain) {
    reg.f64(3, n.stat[0]);  // sum_gradients
    reg.f64(4, n.stat[1]);  // sum_hessians
    reg.f64(5, n.stat[2]);  // sum_weights
  } else {
    Pb dist;  // utils.proto.NormalDistributionDouble
    dist.f64(1, n.stat[0]);
    dist.f64(2, n.stat[1]);
    dist.f64(3, n.stat[2]);
    reg.msg(2, dist);
  }
  Pb node;
  node.msg(2, reg);  // Node.regressor
  if (n.feature >= 0) {
    Pb cond;  // Condition
    if (n.condition_type == YGG_FEATURE_CATEGORICAL) {
      // SetPositiveAttributeSetOfCategoricalContainsCondition (learner/decision_tree/utils.cc:31-63):
      // the smaller of a bitmap over the categories and a sorted int32 vector.
      const int num_values = feature_num_values ? feature_num_values[n.feature] : 256;
      const uint32_t* words = set != nullptr ? set : n.cat_mask;
      const int limit = set != nullptr ? num_values : 256;   // categories the set holds
      auto positive = [&](int c) { return ((words[c >> 5] >> (c & 31)) & 1u) != 0; };
      int num_positive = 0;
      for (int c = 0; c < limit; c++) num_positive += positive(c) ? 1 : 0;
      const int64_t usage_bitmap = (num_values + 7) / 8, usage_vector = 4 * static_cast<int64_t>(num_positive);
      if (usage_bitmap <= usage_vector) {
        std::string bitmap(static_cast<size_t>(usage_bitmap), '\0');
        for (int c = 0; c < num_values && c < limit; c++)
          if (positive(c)) bitmap[c / 8] = static_cast<char>(bitmap[c / 8] | (1 << (c & 7)));
        Pb cb;  // Condition.ContainsBitmap
        cb.bytes(1, bitmap);  // elements_bitmap
        cond.msg(5, cb);      // contains_bitmap_condition
      } else {
        Pb packed;
        for (int c = 0; c < limit; c++)
          if (positive(c)) packed.varint(static_cast<uint64_t>(c));
        Pb cv;  // Condition.ContainsVector
        cv.bytes(1, packed.s);  // elements, packed
        cond.msg(4, cv);        // contains_condition
      }
    } else if (n.condition_type == YGG_FEATURE_NUMERICAL) {
      Pb hi;  // Condition.Higher: value >= threshold (a presorted numerical column)
      hi.f32(1, n.threshold_value);  // threshold
      cond.msg(2, hi);               // higher_condition
    } else {
      Pb dh;  // Condition.DiscretizedHigher
      dh.i64(1, n.threshold_bin);
      cond.msg(6, dh);  // discretized_higher_condition
    }
    Pb nc;  // NodeCondition
    nc.i64(1, n.na_value ? 1 : 0);
    nc.i64(2, feature_col_idx[n.feature]);  // attribute = dataspec column index
    nc.msg(3, cond);
    nc.i64(4, n.num_examples);
    nc.f64(5, static_cast<double>(n.num_examples));
    nc.f32(6, n.split_score);
    nc.i64(7, n.num_pos_examples);
    nc.f64(8, static_cast<double>(n.num_pos_examples));
    node.msg(3, nc);
  }
  node.i64(4, n.num_examples);  // num_pos_training_examples_without_weight (= node size, training.cc:4883)
  return node.s;
}

}  // namespace

extern "C" int ygg_model_write_ydf(const ygg_model_desc* d) {
  if (!d || !d->directory || !d->data_spec_pb || !d->feature_col_idx || !d->trees || !d->tree_offsets)
    return YGG_ERR_INVALID_ARGUMENT;
  if (d->num_trees < 0 || d->num_features <= 0) return YGG_ERR_INVALID_ARGUMENT;
  const std::string dir(d->directory);
  if (mkdir(dir.c_str(), 0755) != 0 && errno != EEXIST) return YGG_ERR_IO;

  // ---- header.pb : model::proto::AbstractModel ----
  Pb h;
  h.bytes(1, "GRADIENT_BOOSTED_TREES");                       // name
  h.i64(2, d->task);                                          // task: 1 CLASSIFICATION, 2 REGRESSION
  h.i64(3, d->label_col_idx);                                 // label_col_idx
  for (int i = 0; i < d->num_features; i++) h.i64(5, d->feature_col_idx[i]);  // input_features
  h.i64(6, -1);                                               // ranking_group_col_idx
  h.i64(8, 1);                                                // classification_outputs_probabilities
  h.i64(9, -1);                                               // uplift_treatment_col_idx
  {
    Pb md;  // Metadata
    md.bytes(4, "ygg_b200");  // framework
    h.msg(10, md);
  }
  h.i64(12, 0);                                               // is_pure_model
  if (!write_file(dir + "/header.pb", h.s)) return YGG_ERR_IO;

  // ---- data_spec.pb : provided by the harness (it owns names and boundaries) ----
  if (!write_file(dir + "/data_spec.pb", std::string(reinterpret_cast<const char*>(d->data_spec_pb), d->data_spec_len)))
    return YGG_ERR_IO;

  // ---- gradient_boosted_trees_header.pb ----
  Pb g;
  g.i64(1, 1);                                                // num_node_shards
  g.i64(2, d->num_trees);                                     // num_trees
  const int per_iter = d->num_trees_per_iter > 1 ? d->num_trees_per_iter : 1;
  // Loss: BINOMIAL_LOG_LIKELIHOOD = 1, SQUARED_ERROR = 2, MULTINOMIAL_LOG_LIKELIHOOD = 3
  g.i64(3, d->loss == YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD ? 1 : (d->loss == YGG_LOSS_MULTINOMIAL_LOG_LIKELIHOOD ? 3 : 2));
  for (int k = 0; k < per_iter; k++) g.f32(4, d->initial_prediction);  // initial_predictions (repeated float)
  g.i64(5, per_iter);                                         // num_trees_per_iter
  if (d->has_validation_loss) g.f32(6, d->validation_loss);   // validation_loss
  g.bytes(7, "BLOB_SEQUENCE");                                // node_format
  {
    Pb logs;  // TrainingLogs
    const int n_logs = d->num_log_entries > 0 ? d->num_log_entries : d->num_trees / per_iter;
    for (int i = 0; i < n_logs; i++) {
      Pb e;
      e.i64(1, (i + 1) * per_iter);                           // number_of_trees
      if (d->train_loss) e.f32(2, d->train_loss[i]);          // training_loss
      if (d->train_secondary) e.f32(3, d->train_secondary[i]);  // training_secondary_metrics
      if (d->valid_loss) e.f32(4, d->valid_loss[i]);          // validation_loss
      if (d->valid_secondary) e.f32(5, d->valid_secondary[i]);  // validation_secondary_metrics
      e.f32(7, 1.f);                                          // subsample_factor
      logs.msg(1, e);
    }
    logs.bytes(2, d->loss == YGG_LOSS_SQUARED_ERROR ? "rmse" : "accuracy");  // secondary_metric_names
    logs.i64(3, d->num_trees);                                // number_of_trees_in_final_model
    g.msg(8, logs);
  }
  g.i64(9, 0);                                                // output_logits
  if (d->early_stopping_triggered) g.i64(11, 1);              // early_stopping_triggered
  if (!write_file(dir + "/gradient_boosted_trees_header.pb", g.s)) return YGG_ERR_IO;

  // ---- nodes-00000-of-00001 : blob sequence, version 1, no compression ----
  std::string blob;
  const uint8_t file_header[8] = {'B', 'S', 1, 0, 0, 0, 0, 0};
  blob.append(reinterpret_cast<const char*>(file_header), 8);
  for (int t = 0; t < d->num_trees; t++) {
    for (int64_t i = d->tree_offsets[t]; i < d->tree_offsets[t + 1]; i++) {
      const int64_t so = d->node_set_offset != nullptr ? d->node_set_offset[i] : -1;
      const uint32_t* set = (so >= 0 && d->cat_set_words != nullptr) ? d->cat_set_words + so : nullptr;
      const std::string rec = encode_node(d->trees[i], d->use_hessian_gain, d->feature_col_idx, d->feature_num_values, set);
      const uint32_t len = static_cast<uint32_t>(rec.size());
      blob.append(reinterpret_cast<const char*>(&len), 4);  // little endian on every supported host
      blob.append(rec);
    }
  }
  if (!write_file(dir + "/nodes-00000-of-00001", blob)) return YGG_ERR_IO;
  if (!write_file(dir + "/done", "")) return YGG_ERR_IO;
  return YGG_OK;
}
