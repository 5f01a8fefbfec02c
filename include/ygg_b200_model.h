/*
 * ygg_b200_model.h — model export of libygg_b200.so (host only).
 * model::SaveModel analogue (model/gradient_boosted_trees/gradient_boosted_trees.cc:111-139): writes
 * the 5-file YDF model directory (header.pb, data_spec.pb, gradient_boosted_trees_header.pb,
 * nodes-00000-of-00001 as a blob sequence, done).
 */
#ifndef YGG_B200_MODEL_H_
#define YGG_B200_MODEL_H_

#include <stdint.h>

#include "ygg_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ygg_model_desc {
  const char* directory;
  int32_t task;                    /* model::proto::Task: 1 = CLASSIFICATION, 2 = REGRESSION */
  int32_t loss;                    /* enum ygg_loss */
  int32_t use_hessian_gain;        /* selects which label statistics a node stores */
  float initial_prediction;
  int32_t num_trees;
  const ygg_node* trees;           /* all trees back to back, each in pre-order */
  const int64_t* tree_offsets;     /* [num_trees + 1] */
  int32_t num_features;
  const int32_t* feature_col_idx;  /* engine feature index -> dataspec column index */
  int32_t label_col_idx;
  const uint8_t* data_spec_pb;     /* serialized dataset::proto::DataSpecification */
  int64_t data_spec_len;
  const float* train_loss;         /* [num_trees] or NULL */
  const float* train_secondary;    /* [num_trees] or NULL */
  int32_t num_log_entries;         /* TrainingLogs entries (0 = num_trees); > num_trees after early stopping */
  const float* valid_loss;         /* [num_log_entries] or NULL: TrainingLogs.Entry.validation_loss */
  const float* valid_secondary;    /* [num_log_entries] or NULL */
  int32_t has_validation_loss;     /* Header.validation_loss is set */
  float validation_loss;
  int32_t early_stopping_triggered; /* Header.early_stopping_triggered */
  int32_t num_trees_per_iter;      /* 0 / 1, or K for the multinomial loss (initial predictions: K x initial_prediction) */
  const int32_t* feature_num_values; /* [num_features]: CategoricalSpec.number_of_unique_values of a categorical
                                        feature (sizes Condition.ContainsBitmap); may be NULL without
                                        categorical features */
  const int64_t* node_set_offset;  /* [tree_offsets[num_trees]] or NULL: for a categorical split on a column with more
                                      than 256 values, the offset of its positive set (ceil(num_values / 32) words) in
                                      cat_set_words; -1 for the other nodes, whose set is cat_mask */
  const uint32_t* cat_set_words;
} ygg_model_desc;

int ygg_model_write_ydf(const ygg_model_desc* desc);

#ifdef __cplusplus
}
#endif
#endif /* YGG_B200_MODEL_H_ */
