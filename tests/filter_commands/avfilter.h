/* tests/filter_commands/avfilter.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The libavfilter stand-in of oracle/ffshim plus what runtime commands need: AV_OPT_FLAG_RUNTIME_PARAM,
 * AVFilter.process_command and ff_filter_process_command.  tests/test_reconfigure.py compiles transform360_cuda with this
 * directory ahead of oracle/ffshim on the include path.  The filter includes "avfilter.h" first, so this header is the
 * one that brings in the stand-in, and every later stand-in header finds it already included.
 */
#ifndef T360_FILTER_COMMANDS_AVFILTER_H
#define T360_FILTER_COMMANDS_AVFILTER_H

#define AVFilter T360ShimFilter /* the stand-in's AVFilter, which has no process_command */
#include "ffshim.h"
#undef AVFilter

#define AV_OPT_FLAG_RUNTIME_PARAM (1 << 15)

/* The stand-in's AVFilter with process_command appended.  oracle/ff_driver.c, compiled with the stand-in alone, reads
 * the same filter object through the stand-in's declaration, a prefix of this one. */
typedef struct AVFilter {
  const char* name;
  const char* description;
  int (*init_dict)(struct AVFilterContext* ctx, AVDictionary** options);
  int (*init)(struct AVFilterContext* ctx);
  int (*query_formats)(struct AVFilterContext* ctx);
  int flags_internal;
  void (*uninit)(struct AVFilterContext* ctx);
  int priv_size;
  const AVClass* priv_class;
  const AVFilterPad* inputs;
  const AVFilterPad* outputs;
  int (*process_command)(struct AVFilterContext* ctx, const char* cmd, const char* arg, char* res, int res_len, int flags);
} AVFilter;

/* av_opt_set for the option types the filters use: numbers (range-checked), named constants of the option's unit.  The
 * target is written only when the value is accepted. */
static inline int ffcmd_opt_set(void* priv, const AVOption* table, const AVOption* o, const char* value) {
  char* end = NULL;
  double v = strtod(value, &end);
  if (end == value || *end) { /* a named constant of the option's unit */
    const AVOption* c = table;
    for (; c->name; c++)
      if (c->type == AV_OPT_TYPE_CONST && o->unit && c->unit && !strcmp(c->unit, o->unit) && !strcmp(c->name, value)) break;
    if (!c->name) return AVERROR(EINVAL);
    v = (double)c->default_val.i64;
  }
  if (v < o->min || v > o->max) return AVERROR(ERANGE);
  uint8_t* dst = (uint8_t*)priv + o->offset;
  if (o->type == AV_OPT_TYPE_FLOAT) *(float*)dst = (float)v;
  else if (o->type == AV_OPT_TYPE_INT) *(int*)dst = (int)v;
  else return AVERROR(EINVAL);
  return 0;
}

/* libavfilter's generic command handler: sets an option of the filter's private context if the option is marked
 * AV_OPT_FLAG_RUNTIME_PARAM; any other name is ENOSYS. */
static inline int ff_filter_process_command(AVFilterContext* ctx, const char* cmd, const char* arg, char* res, int res_len, int flags) {
  (void)res; (void)res_len; (void)flags;
  const AVOption* table = ctx->av_class ? ctx->av_class->option : NULL;
  for (const AVOption* o = table; o && o->name; o++)
    if (o->type != AV_OPT_TYPE_CONST && !strcmp(o->name, cmd))
      return (o->flags & AV_OPT_FLAG_RUNTIME_PARAM) ? ffcmd_opt_set(ctx->priv, table, o, arg) : AVERROR(ENOSYS);
  return AVERROR(ENOSYS);
}

#endif
